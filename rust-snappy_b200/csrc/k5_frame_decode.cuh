// k5_frame_decode.cuh -- K5: device-resident Snappy frame decode.
//
// Replaces reference src/read.rs:104-239 (FrameDecoder::read: the chunk state machine, checksum verification) for a
// frame stream that already sits in device memory; the per-chunk payload decode is K2 (k2_decompress.cuh) and the
// checksum is K3's warp CRC, both run by the same warp while the chunk's output is still in L2.
//
//   k7         (no caller index): builds the chunk index of a clean stream in parallel (k7_frame_index.cuh) into
//              `ooff`, or declines; its count stays on the device (`index_count`).
//   k5_parse   (with a chunk index: the caller's, e.g. the one the frame encoder emits, or K7's): one thread per chunk
//              validates the header, reads the checksum and the decompressed length. Anything unusual -- including a
//              declined K7 index -- raises `need_serial`.
//   k5_walk    (need_serial): one thread walks the chunk headers in stream order exactly like the
//              reference's reader, including its quirk that decompress_len() sees the persistent source buffer
//              (src/read.rs:216) -- ~1 us per chunk, since every header is a dependent global load.
//   scan       output offset of every chunk (generic scan of k4_frame.cuh)
//   k5_decode  warp per chunk: K2 decode or plain copy, then the masked CRC-32C of the produced bytes against the
//              header's (Error::Checksum, src/read.rs:189-196 / :226-233)
//   k5_finish  first failing chunk in stream order -> result {status, bytes produced before it}
#pragma once
#include "common.cuh"
#include "k2_decompress.cuh"
#include "k3_crc32c.cuh"
#include "k4_frame.cuh"

namespace sbk {

static const uint32_t K5_MAX_CBLOCK = 76490;    // reference src/frame.rs:12 (MAX_COMPRESS_BLOCK_SIZE)

struct FChunk { uint64_t body_off; uint32_t body_len; uint32_t dlen; uint32_t want_crc; uint32_t type; };
struct DecodeCtl { uint32_t nchunks; uint32_t need_serial; uint64_t produced; sb_error walk_err; uint32_t go; uint32_t first_bad;
                   uint32_t index_count; };

struct DecodePlan {
    const uint8_t* in; uint64_t n;             // frame stream (device)
    const uint64_t* index; uint32_t index_n;   // optional: offset of every chunk header; index[index_n] = n
    const uint32_t* index_count;               // set: index_n is read here on the device (K7), SB_FRAME_NOT_INDEXABLE = none
    uint32_t fragment;                         // 1: no stream identifier expected (a rank's shard of a stream)
    FChunk* chunks; uint32_t cap_chunks;
    uint64_t* ooff;                            // cap_chunks + 1
    uint64_t* tiles;
    sb_error* statuses;                        // cap_chunks
    DecodeCtl* ctl;
    uint8_t* out; uint64_t cap;
    sb_frame_result* result;
};

SB_DEVICE void k5_set(sb_error* e, uint32_t code, uint64_t a = 0, uint64_t b = 0) { e->code = code; e->_pad = 0; e->a = a; e->b = b; e->c = 0; }

// varint over at most 16 bytes (reference src/bytes.rs:73-90): returns header length, 0 = malformed
SB_DEVICE uint32_t k5_varint(const uint8_t* p, uint32_t n, uint64_t* out) {
    uint64_t v = 0;
    unsigned shift = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (shift >= 64) return 0;
        const uint32_t b = p[i];
        if (b < 0x80) { *out = v | ((uint64_t)b << shift); return i + 1; }
        v |= (uint64_t)(b & 0x7F) << shift;
        shift += 7;
    }
    return 0;
}

// The chunk whose header is at `at` of in[0..n), given the next header at `next` (an index entry pair): a data chunk
// (type 0/1, 4 <= len <= 76490, a stored body of at most 65536 bytes, a varint of at most 65536 within the body's first
// 10 bytes) that ends exactly at `next`. *c = its record; false for anything else (the caller walks the stream).
SB_DEVICE bool k5_check_chunk(const uint8_t* in, uint64_t n, uint64_t at, uint64_t next, FChunk* c) {
    bool ok = at + 8 <= n && next > at && next <= n;
    c->body_off = 0; c->body_len = 0; c->dlen = 0; c->want_crc = 0; c->type = 0;
    if (ok) {
        const uint8_t* h = in + at;
        const uint32_t ty = h[0], len = (uint32_t)h[1] | ((uint32_t)h[2] << 8) | ((uint32_t)h[3] << 16);
        ok = (ty == 0 || ty == 1) && len >= 4 && len <= K5_MAX_CBLOCK && at + 4 + len == next;
        if (ok) {
            c->type = ty;
            c->want_crc = (uint32_t)h[4] | ((uint32_t)h[5] << 8) | ((uint32_t)h[6] << 16) | ((uint32_t)h[7] << 24);
            c->body_off = at + 8; c->body_len = len - 4;
            if (ty == 1) { ok = c->body_len <= kMaxBlock; c->dlen = c->body_len; }
            else {
                uint64_t v = 0;
                const uint32_t hl = k5_varint(h + 8, c->body_len < 10 ? c->body_len : 10, &v);
                ok = hl != 0 && v <= kMaxBlock;
                c->dlen = (uint32_t)v;
            }
        }
    }
    return ok;
}

// ---- parallel header parse over a caller-provided chunk index (clean streams only; anything else -> need_serial)
SB_DEVICE void k5_parse_body(const DecodePlan& p) {
    const uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx();
    DecodeCtl* ctl = p.ctl;
    const uint32_t index_n = p.index_count ? *p.index_count : p.index_n;
    if (index_n == SB_FRAME_NOT_INDEXABLE) {                           // K7 declined: the walk decodes the stream
        if (i == 0) { ctl->need_serial = 1; ctl->nchunks = 0; }
        return;
    }
    if (i == 0) {
        bool ok = index_n <= p.cap_chunks && p.index[index_n] == p.n;
        const uint64_t first = index_n ? p.index[0] : p.n;
        if (p.fragment) ok = ok && first == 0;
        else {
            ok = ok && first == 10 && p.n >= 10;
            if (ok) { const uint8_t id[10] = {0xFF, 6, 0, 0, 's', 'N', 'a', 'P', 'p', 'Y'}; for (int k = 0; k < 10; k++) ok = ok && p.in[k] == id[k]; }
        }
        if (!ok) ctl->need_serial = 1;
        ctl->nchunks = index_n <= p.cap_chunks ? index_n : 0;
    }
    if (i >= index_n || i >= p.cap_chunks) return;
    FChunk c;
    if (!k5_check_chunk(p.in, p.n, p.index[i], p.index[i + 1], &c)) { ctl->need_serial = 1; c.dlen = 0; }
    p.chunks[i] = c;
}

// ---- serial walk of in[0..n) by one thread: exactly the reader's control flow (src/read.rs:111-237), including its
// quirk that decompress_len() sees the persistent source buffer (src/read.rs:216). Every data chunk up to the first
// error goes to sink(i, chunk), at most cap_chunks of them (then SB_E_INVALID{cap_chunks, 1}: chunk table too small).
// Returns the chunk count; *err = the reader's first error (or Ok), *out_produced = the chunks' decompressed bytes.
// Every chunk type advances pos by 4 + its length, so the walk visits a prefix of the stream's header chain.
template <class Sink>
SB_DEVICE uint32_t k5_walk(const uint8_t* in, uint64_t n, bool fragment, uint32_t cap_chunks, Sink sink, sb_error* err,
                           uint64_t* out_produced) {
    uint8_t shadow[16];                                              // first bytes of the reader's persistent `src` buffer
    for (int k = 0; k < 16; k++) shadow[k] = 0;
    sb_error werr;
    k5_set(&werr, SB_OK);
    uint64_t pos = 0, produced = 0;
    uint32_t count = 0;
    bool seen_ident = fragment;
    while (pos < n) {
        if (n - pos < 4) { k5_set(&werr, SB_IO_UNEXPECTED_EOF); break; }
        const uint8_t* h = in + pos;
        for (int k = 0; k < 4; k++) shadow[k] = h[k];
        pos += 4;
        const uint32_t ty = h[0];
        if (!seen_ident) {
            if (ty != 0xFF) { k5_set(&werr, SB_STREAM_HEADER, ty); break; }
            seen_ident = true;
        }
        const uint64_t len = (uint64_t)h[1] | ((uint64_t)h[2] << 8) | ((uint64_t)h[3] << 16);
        if (len > K5_MAX_CBLOCK) { k5_set(&werr, SB_UNSUPPORTED_CHUNK_LENGTH, len, 0); break; }
        if (ty >= 0x02 && ty <= 0x7F) { k5_set(&werr, SB_UNSUPPORTED_CHUNK_TYPE, ty); break; }
        if ((ty >= 0x80 && ty <= 0xFD) || ty == 0xFE) {                   // skippable / padding
            if (n - pos < len) { k5_set(&werr, SB_IO_UNEXPECTED_EOF); break; }
            for (uint64_t k = 0; k < len && k < 16; k++) shadow[k] = in[pos + k];
            pos += len;
        } else if (ty == 0xFF) {
            if (len != 6) { k5_set(&werr, SB_UNSUPPORTED_CHUNK_LENGTH, len, 1); break; }
            if (n - pos < 6) { k5_set(&werr, SB_IO_UNEXPECTED_EOF); break; }
            const uint8_t id[6] = {'s', 'N', 'a', 'P', 'p', 'Y'};
            bool same = true;
            uint64_t a = 0;
            for (int k = 0; k < 6; k++) { shadow[k] = in[pos + k]; same = same && in[pos + k] == id[k]; a |= (uint64_t)in[pos + k] << (8 * k); }
            if (!same) { k5_set(&werr, SB_STREAM_HEADER_MISMATCH, a); break; }
            pos += 6;
        } else {
            if (len < 4) { k5_set(&werr, SB_UNSUPPORTED_CHUNK_LENGTH, len, 0); break; }
            if (n - pos < 4) { k5_set(&werr, SB_IO_UNEXPECTED_EOF); break; }
            const uint32_t want = (uint32_t)in[pos] | ((uint32_t)in[pos + 1] << 8) | ((uint32_t)in[pos + 2] << 16) | ((uint32_t)in[pos + 3] << 24);
            pos += 4;
            const uint32_t body = (uint32_t)len - 4;
            FChunk c;
            c.body_off = pos; c.body_len = body; c.dlen = 0; c.want_crc = want; c.type = ty;
            if (ty == 0x01) {
                if (body > kMaxBlock) { k5_set(&werr, SB_UNSUPPORTED_CHUNK_LENGTH, body, 0); break; }
                if (n - pos < body) { k5_set(&werr, SB_IO_UNEXPECTED_EOF); break; }
                c.dlen = body;
            } else {
                if (n - pos < body) { k5_set(&werr, SB_IO_UNEXPECTED_EOF); break; }
                uint8_t head[16];
                const uint32_t fresh = body < 16 ? body : 16;
                for (uint32_t k = 0; k < 16; k++) head[k] = k < fresh ? in[pos + k] : shadow[k];
                uint64_t v = 0;
                const uint32_t hl = k5_varint(head, 16, &v);
                if (hl == 0) { k5_set(&werr, SB_HEADER); break; }
                if (v > kMaxInput) { k5_set(&werr, SB_TOO_BIG, v, kMaxInput); break; }
                if (v > kMaxBlock) { k5_set(&werr, SB_UNSUPPORTED_CHUNK_LENGTH, v, 0); break; }
                c.dlen = (uint32_t)v;
                for (uint32_t k = 0; k < fresh; k++) shadow[k] = in[pos + k];
            }
            pos += body;
            if (count >= cap_chunks) { k5_set(&werr, SB_E_INVALID, cap_chunks, 1); break; }   // chunk table too small
            sink(count++, c);
            produced += c.dlen;
        }
    }
    *err = werr;
    *out_produced = produced;
    return count;
}

// thread 0 of one warp
SB_DEVICE void k5_walk_body(const DecodePlan& p) {
    DecodeCtl* ctl = p.ctl;
    if (thread_idx() != 0 || block_idx() != 0) return;
    if (p.index && !ctl->need_serial) return;                        // the parallel parse was enough
    FChunk* chunks = p.chunks;
    sb_error werr;
    uint64_t produced;
    ctl->nchunks = k5_walk(p.in, p.n, p.fragment != 0, p.cap_chunks, [&](uint32_t i, const FChunk& c) { chunks[i] = c; },
                           &werr, &produced);
    ctl->walk_err = werr;
    ctl->produced = produced;                                         // provisional (the scan recomputes it)
}

SB_DEVICE void k5_scan_local_body(const DecodePlan& p) {
    const uint32_t count = p.ctl->nchunks;
    if ((uint64_t)block_idx() * K4_TILE >= count && block_idx() != 0) { if (thread_idx() == 0) p.tiles[block_idx()] = 0; return; }
    const FChunk* ch = p.chunks;
    scan_local_body(count, [&](uint32_t i) { return ch[i].dlen; }, p.ooff, p.tiles);
}
SB_DEVICE void k5_scan_tiles_body(const DecodePlan& p) {
    const uint32_t count = p.ctl->nchunks;
    scan_tiles_body(count, 0, p.tiles);
    if (thread_idx() == 0) {
        const uint64_t total = p.tiles[(count + K4_TILE - 1) / K4_TILE];
        p.ctl->produced = total;
        p.ctl->go = total <= p.cap ? 1u : 0u;
        p.ctl->first_bad = 0xFFFFFFFFu;
    }
}

// One chunk by the calling warp: K2 decode or plain copy of its body to dst, then the masked CRC-32C of the produced
// bytes against the header's (Error::Checksum, src/read.rs:189-196 / :226-233). *st = the chunk's status; returns its code.
SB_DEVICE uint32_t k5_decode_chunk(const uint32_t* tab, uint32_t* elems, const FChunk& c, const uint8_t* in, uint8_t* dst,
                                   sb_error* st) {
    uint32_t code = SB_OK;
    if (c.type == 0) code = k2_decode_stream(in + c.body_off, c.body_len, dst, c.dlen, st, nullptr, elems);
    else { warp_copy(dst, in + c.body_off, c.body_len); if (lane_id() == 0) k5_set(st, SB_OK); }
    syncwarp();
    if (code == SB_OK) {
        const uint32_t got = k3_warp_crc32c_masked(tab, dst, c.dlen);
        if (got != c.want_crc) { code = SB_CHECKSUM; if (lane_id() == 0) k5_set(st, SB_CHECKSUM, c.want_crc, got); }
    }
    return code;
}

// warp per chunk: decode / copy, then verify the checksum while the output is hot in L2
SB_DEVICE void k5_decode_body(const DecodePlan& p) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const DecodeCtl* ctl = p.ctl;
    const uint32_t count = ctl->nchunks;
    if (!ctl->go) return;
    const unsigned wpb = block_dim() >> 5, lane = lane_id();
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t u = (uint64_t)block_idx() * wpb + warp_id(); u < count; u += nwarps) {
        const FChunk c = p.chunks[u];
        const uint64_t off = p.tiles[u / K4_TILE] + p.ooff[u];
        uint8_t* dst = p.out + off;
        const uint32_t code = k5_decode_chunk(tab, elems, c, p.in, dst, &p.statuses[u]);
        if (code != SB_OK && lane == 0) atomic_min(&p.ctl->first_bad, (uint32_t)u);
        syncwarp();
        if (lane == 0) p.ooff[u] = off;                                 // absolute from here on
    }
}

SB_DEVICE void k5_finish_body(const DecodePlan& p) {
    if (thread_idx() != 0 || block_idx() != 0) return;
    const DecodeCtl* ctl = p.ctl;
    sb_frame_result r;
    r.nchunks = ctl->nchunks; r._pad = 0;
    // chunk table too small: the walk stopped early, so `produced` is only a lower bound -- report the table first, so
    // that a caller retries with a larger one before it sizes the output
    if (ctl->walk_err.code == SB_E_INVALID && ctl->walk_err.b == 1) { r.status = ctl->walk_err; r.bytes = 0; }
    else if (!ctl->go) { k5_set(&r.status, SB_BUFFER_TOO_SMALL, p.cap, ctl->produced); r.bytes = 0; }
    else if (ctl->first_bad != 0xFFFFFFFFu) { r.status = p.statuses[ctl->first_bad]; r.bytes = p.ooff[ctl->first_bad]; }
    else { r.status = ctl->walk_err; r.bytes = ctl->produced; }
    *p.result = r;
}

}  // namespace sbk

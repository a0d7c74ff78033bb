// k4_frame.cuh -- K4: frame/stream assembly around K1 (and small utility kernels).
//
// Replaces reference src/frame.rs:62-104 (compress_frame: chunk type decision
// `compressed_len >= n - n/8`, 8-byte header = type, u24 length, masked CRC) and
// the chunk loop of src/write.rs:165-192 for a device-resident input; also the
// block concatenation of Encoder::compress for inputs above 64KB
// (src/compress.rs:128-153).
//
// Stream ordered, no host round trip: K1 compresses every <=64KB chunk into a slot
// (and, for frames, leaves the chunk's masked CRC beside it), then
//   k4_scan_local  : final size of every chunk + exclusive scan inside 1024-chunk tiles
//   k4_scan_tiles  : exclusive scan of the tile totals (one CTA; 4M chunks = 4096 tiles)
//   k4_gather      : header + body of every chunk copied to its final offset, stream prefix
//                    (identifier / varint) and the result record written by the first CTA.
#pragma once
#include "common.cuh"

namespace sbk {

static const uint32_t K4_TILE = 1024;      // chunks per scan tile (= threads of k4_scan_local)

struct FramePlan {
    const uint8_t* in;        // uncompressed input (device)
    uint64_t n;               // total bytes
    const uint8_t* slots;     // K1 output slots, stride kSlotStride
    const uint32_t* clens;    // K1 output length per chunk
    const uint32_t* crcs;     // masked CRC per chunk (frame mode)
    uint32_t nchunks;
    uint32_t frame;           // 1: frame chunks with 8-byte headers; 0: raw block concatenation
    uint32_t head_len;        // bytes in front of chunk 0 (stream identifier / varint), <= 16
    uint8_t head[16];
    uint64_t* offs;           // out: offset of each chunk in the final stream; offs[nchunks] = total
    uint64_t* tiles;          // scratch: one entry per tile (+1)
    uint8_t* out;             // final stream
    uint64_t cap;             // capacity of `out`
    sb_frame_result* result;  // out (device, may be null): status, total bytes, chunk count
};

SB_DEVICE uint32_t k4_chunk_len(uint64_t n, uint32_t i) {
    const uint64_t at = (uint64_t)i * kMaxBlock;
    const uint64_t left = n - at;
    return left > kMaxBlock ? kMaxBlock : (uint32_t)left;
}
// a chunk of n input bytes that compresses to c bytes (varint included) is stored uncompressed (src/frame.rs:85).
// A macro, not a function: K4's kernels then compile to the same code as with the comparison written out.
#define K4_CHUNK_RAW(c, n) ((c) >= (n) - (n) / 8)
// bytes chunk i occupies in the final stream
SB_DEVICE uint32_t k4_chunk_size(const FramePlan& p, uint32_t i) {
    const uint32_t c = p.clens[i];
    if (!p.frame) return c;
    const uint32_t n = k4_chunk_len(p.n, i);
    return 8 + (K4_CHUNK_RAW(c, n) ? n : c);
}

// per-chunk input lengths for K1: all 65536 except the last (src/write.rs:171-174)
SB_DEVICE void k4_fill_lens_body(uint32_t* lens, uint64_t n, uint32_t nchunks) {
    const uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx();
    if (i < nchunks) lens[i] = k4_chunk_len(n, (uint32_t)i);
}

// Generic two-level exclusive scan of `count` u32 values into u64 offsets (tiles of 1024 = one CTA of 1024 threads).
// CTA t: scan of values [1024t, 1024t+1024) -> offs (tile-relative), tile total -> tiles[t]
template <class Val>
SB_DEVICE void scan_local_body(uint32_t count, Val val, uint64_t* offs, uint64_t* tiles) {
    uint32_t* sh = (uint32_t*)smem();      // 32 warp totals
    const unsigned t = thread_idx(), lane = lane_id(), wid = warp_id();
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + t;
    const uint32_t v = i < count ? val((uint32_t)i) : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) { const uint32_t x = shfl_up(incl, k); if (lane >= (unsigned)k) incl += x; }
    if (lane == 31) sh[wid] = incl;
    syncthreads();
    if (wid == 0) {
        uint32_t w = sh[lane], wi = w;
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) { const uint32_t x = shfl_up(wi, k); if (lane >= (unsigned)k) wi += x; }
        sh[lane] = wi - w;
        if (lane == 31) tiles[block_idx()] = wi;
    }
    syncthreads();
    if (i < count) offs[i] = (uint64_t)sh[wid] + (incl - v);
}
// one CTA: exclusive scan of the tile totals in place (+ base), grand total -> tiles[ntiles]
SB_DEVICE void scan_tiles_body(uint32_t count, uint64_t base, uint64_t* tiles) {
    uint64_t* sh = (uint64_t*)smem();      // block_dim entries
    const unsigned t = thread_idx(), nt = block_dim();
    const uint32_t ntiles = (count + K4_TILE - 1) / K4_TILE;
    const uint32_t per = (ntiles + nt - 1) / nt;
    const uint32_t lo = per * t < ntiles ? per * t : ntiles;
    const uint32_t hi = lo + per < ntiles ? lo + per : ntiles;
    uint64_t sum = 0;
    for (uint32_t i = lo; i < hi; i++) sum += tiles[i];
    sh[t] = sum;
    syncthreads();
    if (t == 0) {
        uint64_t run = base;
        for (unsigned k = 0; k < nt; k++) { const uint64_t v = sh[k]; sh[k] = run; run += v; }
        tiles[ntiles] = run;
    }
    syncthreads();
    uint64_t run = sh[t];
    for (uint32_t i = lo; i < hi; i++) { const uint64_t v = tiles[i]; tiles[i] = run; run += v; }
}
SB_DEVICE void k4_scan_local_body(const FramePlan& p) {
    scan_local_body(p.nchunks, [&](uint32_t i) { return k4_chunk_size(p, i); }, p.offs, p.tiles);
}
SB_DEVICE void k4_scan_tiles_body(const FramePlan& p) { scan_tiles_body(p.nchunks, p.head_len, p.tiles); }

// warp per chunk: header + body into the final stream; offs[] becomes absolute
SB_DEVICE void k4_gather_body(const FramePlan& p) {
    const unsigned wpb = block_dim() >> 5, lane = lane_id();
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    const uint32_t ntiles = (p.nchunks + K4_TILE - 1) / K4_TILE;
    const uint64_t total = p.tiles[ntiles];
    const bool fits = total <= p.cap;
    if (block_idx() == 0 && warp_id() == 0) {
        if (fits && lane < p.head_len) p.out[lane] = p.head[lane];
        if (lane == 0) {
            p.offs[p.nchunks] = total;
            if (p.result) {
                sb_frame_result r;
                r.status.code = fits ? SB_OK : SB_BUFFER_TOO_SMALL; r.status._pad = 0;
                r.status.a = fits ? 0 : p.cap; r.status.b = fits ? 0 : total; r.status.c = 0;
                r.bytes = fits ? total : 0; r.nchunks = p.nchunks; r._pad = 0;
                *p.result = r;
            }
        }
    }
    for (uint64_t u = (uint64_t)block_idx() * wpb + warp_id(); u < p.nchunks; u += nwarps) {
        const uint32_t i = (uint32_t)u;
        const uint64_t off = p.tiles[i / K4_TILE] + p.offs[i];
        syncwarp();
        if (lane == 0) p.offs[i] = off;
        if (!fits) continue;
        uint8_t* dst = p.out + off;
        const uint8_t* slot = p.slots + (uint64_t)i * kSlotStride;
        if (p.frame) {
            const uint32_t n = k4_chunk_len(p.n, i), c = p.clens[i];
            const bool raw = K4_CHUNK_RAW(c, n);
            const uint32_t body = raw ? n : c, clen = 4 + body, crc = p.crcs[i];
            if (lane < 8) {
                const uint64_t hdr = (uint64_t)(raw ? 1u : 0u) | ((uint64_t)clen << 8) | ((uint64_t)crc << 32);
                dst[lane] = (uint8_t)(hdr >> (8 * lane));                    // src/frame.rs:91-93
            }
            warp_copy_t<true>(dst + 8, raw ? p.in + (uint64_t)i * kMaxBlock : slot, body);
        } else {
            warp_copy_t<true>(dst, slot, p.clens[i]);
        }
    }
}

// K6: synthetic input -- unit i = text[off_i .. off_i+len), off_i = ((first+i)*mul) % (text_len-len)
struct GenPlan {
    const uint8_t* text; uint64_t text_len; uint8_t* out; uint64_t stride;
    uint32_t len; uint64_t first, count, mul;
};
SB_DEVICE void k6_generate_body(const GenPlan& g) {
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    const uint64_t span = g.text_len - g.len;
    for (uint64_t u = (uint64_t)block_idx() * wpb + warp_id(); u < g.count; u += nwarps) {
        const uint64_t off = span ? ((g.first + u) * g.mul) % span : 0;
        warp_copy(g.out + u * g.stride, g.text + off, g.len);
    }
}

}  // namespace sbk

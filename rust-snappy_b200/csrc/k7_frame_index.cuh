// k7_frame_index.cuh -- K7: chunk index of a frame stream in device memory, built in parallel.
//
// Output: the offset of every chunk header followed by n (exactly the d_chunk_offs layout the frame encoder emits and
// k5_parse consumes), and the chunk count -- or the verdict SB_FRAME_NOT_INDEXABLE. Only clean streams are indexed:
// the 10-byte stream identifier at offset 0 (none for a fragment), then data chunks only (type 0x00/0x01,
// 4 <= len <= 76490, a type-0x01 body of at most 65536 bytes) that cover [s0, n) exactly. Anything else (skippable or
// padding chunks, a repeated identifier, reserved types, truncation, more than max_chunks chunks, a segment whose
// entry chunk is not among the survivors kept) is declined, and the decoder takes its serial walk.
//
// Why this cannot change a decoded byte or an error: chunk headers form a linked list starting at s0, and k5_parse
// checks every index entry against it -- the first entry is s0 (and the identifier bytes are right), every chunk
// satisfies at + 4 + len == next with a valid type and length, and the last entry is n. An index that k5_parse
// accepts is therefore the reader's own walk; K7 only decides whether the parallel parse is taken.
//
// No step is a dependent chain over all chunks. [s0, n) is cut into segments of `seg` bytes (seg >= 128 KiB, more
// than the 76,494 bytes a chunk can span), so the first chunk header at or after segment start b_k lies in the window
// [b_k, b_k + 76494), and every chain leaving segment k lands in segment k+1's window.
//   k7_survivors  warp per segment: lanes test every window position for a plausible data-chunk header, each
//                 candidate is walked (one lane per candidate) until it reaches the segment end (it survives) or meets
//                 an implausible header (it is dropped). The first K7_KEEP survivors in position order are kept as
//                 (entry, exit, chunks). False starts in compressed or random bytes die within a hop or two; one that
//                 lands on a true header joins the true chain and survives with the same exit.
//   k7_stitch     one CTA: e_0 = s0, e_{k+1} = exit of segment k's survivor whose entry is e_k, base_k = running chunk
//                 count. Serial, but one shared-memory step per segment (256 KiB), not per chunk.
//   k7_emit       thread per segment: walks again from e_k and writes index[base_k + j]; index[total] = n.
// The true entry e_k is the FIRST chain header at or after b_k, so it is always among the first survivors: a segment
// is only lost when K7_KEEP false starts before e_k all survive to the segment end.
#pragma once
#include "k5_frame_decode.cuh"

namespace sbk {

static const uint32_t K7_KEEP = 8;                      // survivors kept per segment
static const uint64_t K7_SPAN = 4 + K5_MAX_CBLOCK;      // most bytes one chunk occupies (header + body)
static const uint64_t K7_SEG_MIN = 128u << 10;          // segment length floor (> K7_SPAN)
static const uint64_t K7_SEG_DEFAULT = 256u << 10;
static const unsigned K7_STITCH_THREADS = 256;          // segments resolved per shared-memory tile

// survivors of one segment; offsets relative to the segment start b_k
struct K7Seg { uint32_t entry[K7_KEEP], exit[K7_KEEP], chunks[K7_KEEP]; };
static const size_t K7_STITCH_SMEM = (size_t)K7_STITCH_THREADS * (3 * K7_KEEP + 1) * 4 + 16;

struct IndexPlan {
    const uint8_t* in; uint64_t n;
    uint64_t s0;                       // offset of the first chunk header: 10, or 0 for a fragment
    uint64_t seg;                      // segment length
    uint32_t nseg;
    uint32_t fragment;
    uint32_t max_chunks;
    uint32_t decline;                  // decided on the host (no identifier room, too many chunks for max_chunks, ...)
    K7Seg* segs;                       // nseg
    uint32_t *nsurv, *ent, *base;      // nseg each: survivors kept; e_k - b_k; chunks before segment k
    uint64_t* index;                   // max_chunks + 1
    uint32_t* count;                   // chunks, or SB_FRAME_NOT_INDEXABLE
};

// Segment length for `body` bytes of chunks when the survivor table holds at most `max_segs` segments (0: none fits).
inline uint64_t k7_seg_len(uint64_t body, uint64_t max_segs, uint64_t want) {
    if (max_segs == 0) return 0;
    uint64_t g = want < K7_SEG_MIN ? K7_SEG_MIN : want;
    const uint64_t need = (body + max_segs - 1) / max_segs;
    if (g < need) g = (need + 4095) / 4096 * 4096;
    return g > (1ull << 31) ? 0 : g;   // offsets inside a segment stay 32-bit
}

// segs: room for max_segs survivor records; meta: 3 * max_segs words
inline IndexPlan k7_make_plan(const uint8_t* in, uint64_t n, uint32_t fragment, uint32_t max_chunks, uint64_t want_seg,
                              K7Seg* segs, uint64_t max_segs, uint32_t* meta, uint64_t* index, uint32_t* count) {
    IndexPlan p;
    memset(&p, 0, sizeof p);
    p.in = in; p.n = n; p.fragment = fragment ? 1u : 0u; p.max_chunks = max_chunks;
    p.s0 = fragment ? 0 : 10;
    const uint64_t body = n > p.s0 ? n - p.s0 : 0;
    p.seg = k7_seg_len(body, max_segs, want_seg);
    // a clean stream needs at least ceil(body / K7_SPAN) chunks
    p.decline = (n < p.s0 || p.seg == 0 || (body + K7_SPAN - 1) / K7_SPAN > max_chunks) ? 1u : 0u;
    p.nseg = p.decline ? 0 : (uint32_t)((body + p.seg - 1) / p.seg);
    p.segs = segs; p.nsurv = meta; p.ent = meta + max_segs; p.base = meta + 2 * max_segs;
    p.index = index; p.count = count;
    return p;
}

// The decoder's own scratch: the index goes where the scan's output offsets go later (k5_parse reads it first), the
// survivor table over the status records and the per-segment words over the chunk table (both written after K7).
inline IndexPlan k7_plan_for_decode(const DecodePlan& d, uint64_t want_seg) {
    const uint64_t max_segs = (uint64_t)d.cap_chunks * sizeof(sb_error) / sizeof(K7Seg);
    return k7_make_plan(d.in, d.n, d.fragment, d.cap_chunks, want_seg, (K7Seg*)d.statuses, max_segs,
                        (uint32_t*)d.chunks, d.ooff, &d.ctl->index_count);
}

// Data-chunk header at p that stays inside the stream: *next = the following header
SB_DEVICE bool k7_hop(const uint8_t* in, uint64_t n, uint64_t p, uint64_t* next) {
    if (n - p < 8) return false;
    const uint32_t ty = in[p], len = (uint32_t)in[p + 1] | ((uint32_t)in[p + 2] << 8) | ((uint32_t)in[p + 3] << 16);
    if (ty > 1 || len < 4 || len > K5_MAX_CBLOCK || (ty == 1 && len - 4 > kMaxBlock) || n - p - 4 < len) return false;
    *next = p + 4 + len;
    return true;
}

// segment k < p.nseg of a stream that is not declined, by the calling warp
SB_DEVICE void k7_survivors_seg(const IndexPlan& p, uint64_t k) {
    const unsigned lane = lane_id();
    const uint8_t* in = p.in;
    const uint64_t n = p.n, b = p.s0 + k * p.seg;
    const uint64_t lim = b + p.seg < n ? b + p.seg : n;
    const uint64_t wend = k == 0 ? b + 1 : (b + K7_SPAN < n ? b + K7_SPAN : n);   // segment 0 starts at s0 itself
    K7Seg* rec = &p.segs[k];
    uint32_t kept = 0;
    for (uint64_t w = b; w < wend && kept < K7_KEEP; w += 32 * 8) {
        uint32_t cmask = 0;                                          // bit j: position w + 32j + lane is a candidate
#pragma unroll
        for (int j = 0; j < 8; j++) {                                // 16 independent coalesced byte loads per lane
            const uint64_t q = w + 32 * j + lane;
            const uint32_t t0 = q < wend ? in[q] : 0xFF, t3 = q < wend && q + 3 < n ? in[q + 3] : 0xFF;
            cmask |= (t0 <= 1 && t3 <= 1 ? 1u : 0u) << j;           // type 0/1 and len < 2^17
        }
#pragma unroll 1
        for (int j = 0; j < 8 && kept < K7_KEEP; j++) {
            const uint64_t q = w + 32 * j + lane;
            const bool cand = (cmask >> j) & 1u;
            if (!any(cand)) continue;
            bool alive = cand;
            uint64_t at = q;
            uint32_t hops = 0;
            while (alive && at < lim) {
                uint64_t nx = at;
                alive = k7_hop(in, n, at, &nx);
                at = nx; hops++;
            }
            const uint32_t surv = ballot(alive);
            const uint32_t slot = kept + popc(surv & ((1u << lane) - 1u));
            if (alive && slot < K7_KEEP) {
                rec->entry[slot] = (uint32_t)(q - b); rec->exit[slot] = (uint32_t)(at - b); rec->chunks[slot] = hops;
            }
            kept += popc(surv);
        }
    }
    if (lane == 0) p.nsurv[k] = kept < K7_KEEP ? kept : K7_KEEP;
}
SB_DEVICE void k7_survivors_body(const IndexPlan& p) {
    const uint64_t k = (uint64_t)block_idx() * (block_dim() >> 5) + warp_id();
    if (p.decline || k >= p.nseg) return;
    k7_survivors_seg(p, k);
}

SB_DEVICE void k7_stitch_body(const IndexPlan& p) {
    const unsigned T = K7_STITCH_THREADS, t = thread_idx();
    uint32_t* sE = (uint32_t*)smem();
    uint32_t* sX = sE + T * K7_KEEP;
    uint32_t* sC = sX + T * K7_KEEP;
    uint32_t* sN = sC + T * K7_KEEP;
    uint32_t* sOk = sN + T;
    uint64_t e = p.s0, total = 0;                                    // thread 0's chain state
    bool ok = !p.decline;
    if (t == 0) {
        if (ok && !p.fragment) {
            const uint8_t id[10] = {0xFF, 6, 0, 0, 's', 'N', 'a', 'P', 'p', 'Y'};
            for (int i = 0; i < 10; i++) ok = ok && p.in[i] == id[i];
        }
        sOk[0] = ok;
    }
    syncthreads();
    for (uint64_t k0 = 0; k0 < p.nseg; k0 += T) {
        if (!sOk[0]) break;
        const uint64_t k = k0 + t;
        if (k < p.nseg) {                                            // independent loads of this tile's survivors
            const uint32_t m = p.nsurv[k];
            sN[t] = m;
            for (uint32_t i = 0; i < m; i++) {
                sE[t * K7_KEEP + i] = p.segs[k].entry[i]; sX[t * K7_KEEP + i] = p.segs[k].exit[i]; sC[t * K7_KEEP + i] = p.segs[k].chunks[i];
            }
        }
        syncthreads();
        if (t == 0) {
            for (uint32_t j = 0; j < T && k0 + j < p.nseg && ok; j++) {
                const uint64_t b = p.s0 + (k0 + j) * p.seg;
                const uint32_t rel = (uint32_t)(e - b);
                p.ent[k0 + j] = rel; p.base[k0 + j] = (uint32_t)total;
                if (e == p.n) continue;                              // the last chunk ended inside the previous segment
                int hit = -1;
#pragma unroll
                for (int i = 0; i < (int)K7_KEEP; i++) if ((uint32_t)i < sN[j] && sE[j * K7_KEEP + i] == rel) hit = i;
                if (hit < 0) { ok = false; break; }
                total += sC[j * K7_KEEP + hit];
                e = b + sX[j * K7_KEEP + hit];
                ok = total <= p.max_chunks;
            }
            sOk[0] = ok;
        }
        syncthreads();
    }
    if (t == 0) *p.count = ok && e == p.n ? (uint32_t)total : (uint32_t)SB_FRAME_NOT_INDEXABLE;
}

// the index entries of the chunks of segment k < p.nseg of an indexed stream
SB_DEVICE void k7_emit_seg(const IndexPlan& p, uint64_t k) {
    const uint64_t b = p.s0 + k * p.seg;
    const uint64_t lim = b + p.seg < p.n ? b + p.seg : p.n;
    uint64_t at = b + p.ent[k];
    uint32_t j = p.base[k];
    while (at < lim) {                                               // the survivor walk already checked every hop
        p.index[j++] = at;
        at += 4 + ((uint32_t)p.in[at + 1] | ((uint32_t)p.in[at + 2] << 8) | ((uint32_t)p.in[at + 3] << 16));
    }
}
SB_DEVICE void k7_emit_body(const IndexPlan& p) {
    const uint64_t k = (uint64_t)block_idx() * block_dim() + thread_idx();
    const uint32_t total = *p.count;
    if (total == SB_FRAME_NOT_INDEXABLE) return;
    if (k == 0) p.index[total] = p.n;
    if (k >= p.nseg) return;
    k7_emit_seg(p, k);
}

}  // namespace sbk

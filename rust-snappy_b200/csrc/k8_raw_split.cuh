// k8_raw_split.cuh -- K8: decode one large raw stream in parallel by finding the compressed start of every 64 KB block.
//
// Every encoder that matters (the reference, src/compress.rs:99-154; our K1; Google's C++ snappy) compresses a raw
// stream in independent 65,536-byte blocks: no element crosses an output position that is a multiple of 65,536, and no
// copy reaches back before its block's first byte. Only the blocks' compressed start offsets are unknown. K8 finds them
// as a cut table cut[0..B]: cut[j] is the offset of the element that starts at output position 65536*j, cut[0] is the
// end of the varint header, cut[B] = n, B = ceil(dn / 65536). Then one warp per block decodes [cut[j], cut[j+1]) with
// K2's element loop and block-local bounds. Anything K8 cannot split this way is declined, and one warp decodes the
// whole stream exactly as before (k8_fallback).
//
// The stream is cut into segments of `seg` compressed bytes (seg >= 128 KiB, more than the longest element the parallel
// path accepts: a literal of at most 65,536 bytes and its 5-byte tag). Snappy elements resynchronise: two parses that
// reach the same byte agree from there on.
//   k8_header    one thread: varint header; malformed, too big or over `cap` -> decline.
//   k8_chains    warp per segment: the "canonical" parse from the segment start b_k (the true start for segment 0)
//                with K2's 32-byte speculative window (k2_window.inc), output-free; marks every element start below
//                the segment end in a bitmap and records the exit X_k, the first element start at or after the end.
//                A parse that reaches an element no split stream has (a literal over 64 KB, an element past the end)
//                is dropped and restarted at the next byte.
//   k8_merge     warp per segment k >= 1: parses the true chain from X_{k-1} (what segment k's true entry is whenever
//                segment k-1's true parse merged with its canonical one) with the same window step until it reaches a
//                marked start (from there it is the canonical chain, so its exit is X_k) or leaves the segment (its
//                own last position). Copy-dense text can take tens of thousands of elements to merge.
//   k8_stitch    one CTA: e_0 = header end; e_{k+1} = exit of segment k from the true entry e_k, which is k8_merge's
//                result when e_k == X_{k-1}, else a walk of one thread from e_k of at most K8_HOPS elements. One
//                shared-memory step per segment where the speculation held.
//   k8_counts    warp per segment: output bytes of the true elements in [e_k, exit_k) -> K4's generic two-level scan.
//   k8_cuts      warp per segment: re-parses [e_k, exit_k) from its output offset and records cut[j] at every multiple
//                of 65,536; an element that straddles one, or a total other than dn, declines.
//   k8_blocks    warp per block: K2 over the block alone (k2_decode_stream<false>); any status but Ok declines.
//   k8_fallback  one warp, always enqueued: writes the result, or -- when declined -- runs K2 over the whole stream.
//
// Why the result is exactly the reference's: parsing is deterministic and segment 0 starts at the true start, so by
// induction every accepted exit, and so every cut, is an element boundary of the reference's own parse. A block that
// decodes Ok with block-local bounds also passes the reference's global checks, which are weaker: its copy offsets are
// at most the local output position (<= the global one), and its literal and copy bounds lie inside the block, so
// inside the stream. "All blocks Ok, cuts cover [header end, n), lengths sum to dn" therefore implies that the
// reference returns Ok with the same bytes. Everything else (copies into an earlier block, elements straddling a
// block boundary, literals over 64 KB, parses that never merge, every corrupt or truncated stream) is decoded by the
// one-warp K2 path, so errors keep today's variant and payload.
#pragma once
#include "k2_decompress.cuh"
#include "k4_frame.cuh"

namespace sbk {

static const uint64_t K8_SEG_MIN = 128u << 10;          // segment length floor (> 65541, the longest accepted element)
static const uint64_t K8_SEG_MAX = 64u << 20;           // keeps a segment's output below 2^32 (at most 22 bytes per byte)
static const uint64_t K8_SEG_DEFAULT = 128u << 10;
// Elements one thread of the stitch walks in a segment whose true entry is not where k8_merge started (the previous
// segment's true parse never met its canonical one) before it declines. That happens with 64 KB literals, which a
// segment holds only a few of; a parse that does not merge within this many hops (1-byte literals whose parity never
// lines up: 65,536 hops per segment) is left to the one-warp decoder rather than walked serially.
static const uint32_t K8_HOPS = 1024;
static const uint64_t K8_BAD = ~0ull;                   // "no valid exit": the stream is declined
static const uint64_t K8_MET = ~1ull;                   // k8_walk<.., kMeet>: reached a start of the canonical parse
static const uint32_t K8_MAX_BLOCKS = 65536;            // output < 2^32
static const unsigned K8_STITCH_THREADS = 256;

struct RawCtl { uint64_t dn; uint32_t hl, nblk, decline, out_len; };

struct RawPlan {
    const uint8_t* in; uint64_t n;     // the raw stream (device), n < 2^32
    uint8_t* out; uint64_t cap;
    sb_frame_result* result;
    uint64_t seg; uint32_t nseg;
    RawCtl* ctl;
    uint32_t* marks;                   // bit p: p is an element start of its segment's canonical parse (zeroed)
    uint64_t *X, *Y, *ent, *ext;       // nseg each: canonical exit, merged exit from X_{k-1}, true entry, true exit
    uint32_t* cnt;                     // nseg: output bytes of each segment
    uint64_t *offs, *tiles;            // scan of cnt
    uint32_t* cut;                     // K8_MAX_BLOCKS + 1
};

// Segment length for a request (0: the default): the floor, and no more segments than the scratch was sized for.
inline uint64_t k8_seg_len(uint64_t want) {
    const uint64_t g = want ? want : K8_SEG_DEFAULT;
    return g < K8_SEG_MIN ? K8_SEG_MIN : g > K8_SEG_MAX ? K8_SEG_MAX : (g + 31) / 32 * 32;
}
inline uint64_t k8_max_segs(uint64_t n) { return n / K8_SEG_MIN + 2; }

// Whether the stream is declined, the same for every lane of the warp: k8_cuts and k8_blocks set the flag while other
// warps of the same launch read it, and a warp whose lanes disagreed would split around its warp collectives.
SB_DEVICE bool k8_declined(const RawPlan& p) { return shfl(ld_volatile(&p.ctl->decline), 0) != 0; }

// the element at p (< n): *next = the byte after it. False when it runs past n or is a literal longer than a block.
SB_DEVICE bool k8_hop(const uint8_t* in, uint64_t n, uint64_t p, uint64_t* next) {
    const uint32_t tag = in[p], kind = tag & 3u;
    uint64_t hdr, len = 0;
    if (kind == 0) {
        const uint32_t L = tag >> 2;
        if (L < 60) { hdr = 1; len = L + 1; }
        else {
            const uint32_t nb = L - 59;
            hdr = 1 + nb;
            if (n - p < hdr) return false;
            for (uint32_t i = 0; i < nb; i++) len |= (uint64_t)in[p + 1 + i] << (8 * i);
            len += 1;
        }
    } else hdr = kind == 1 ? 2 : kind == 2 ? 3 : 5;
    if (len > kMaxBlock || n - p < hdr + len) return false;
    *next = p + hdr + len;
    return true;
}

// Walk of the true chain of segment k from e (an element start >= b_k): its exit.
SB_DEVICE uint64_t k8_resolve(const RawPlan& p, uint64_t k, uint64_t e) {
    const uint64_t lim = (k + 1) * p.seg < p.n ? (k + 1) * p.seg : p.n;
    uint64_t at = e;
    for (uint32_t hops = 0; at < lim; hops++) {
        if ((p.marks[at >> 5] >> (at & 31u)) & 1u) return p.X[k];   // joined the canonical parse
        if (hops == K8_HOPS || !k8_hop(p.in, p.n, at, &at)) return K8_BAD;
    }
    return at;
}

// Parse-only walk of the warp over the element starts in [s0, stop) (s0 an element start, stop <= n) with K2's window
// step. Returns the first element start >= stop, or K8_BAD when an element runs past n, is a literal longer than a
// block, or (kCut) straddles a block boundary. *out = output bytes of the elements walked. kMark (the canonical parse
// of a segment, from a byte that need not be an element start): set the bits of its element starts in `marks`, and on
// such an element drop the marks of the parse so far and start again at the next byte, so that the marks always lie
// on the one parse that ends at the returned exit. kMeet: return K8_MET at the first element start that is marked.
// kCut: record cut[j] for every element at global output position 65536*j < dn, with obase the output position of the
// element at s0.
template <bool kMark, bool kCut, bool kMeet = false>
SB_DEVICE uint64_t k8_walk(const RawPlan& p, uint64_t s0, uint64_t stop, uint64_t obase, uint64_t dn, uint64_t* out) {
    const unsigned lane = lane_id();
    const uint8_t* in = p.in;
    const uint8_t* in_end = p.in + p.n;
    const uint8_t* src = p.in;
    const uint32_t sn = (uint32_t)p.n;
    uint32_t s = (uint32_t)s0, piece = s;                            // piece: where the current canonical parse began
    uint64_t d = 0;
    while (s < stop) {
#include "k2_window.inc"
        (void)off; (void)spill; (void)E; (void)valid;
        const uint64_t lim = stop - s;                                  // <= rem
        const bool mine = ((M >> lane) & 1u) && lane < lim;             // lane 0 always is
        const uint64_t end = (uint64_t)lane + hdr + (kind == 0 ? len : 0);
        const uint32_t inm = ballot(mine);
        const uint32_t bad = ballot(mine && (end > rem || (kind == 0 && len > kMaxBlock)));
        if (bad) {
            if (!kMark) return K8_BAD;
            // A parse that starts inside an element soon merges with the true one, or reaches an element that cannot
            // be part of a valid split stream (mostly a literal "longer" than a block). Then it is no chain at all:
            // its marks go, and the canonical parse starts again at the next byte.
            const uint32_t q = s + (ffs(bad) - 1);
            syncwarp();                                              // lane 0's marks are visible to every lane
            for (uint32_t w = (piece >> 5) + lane; piece < s && w <= ((s - 1) >> 5); w += 32) {
                const uint32_t lo = w << 5 < piece ? piece - (w << 5) : 0u;
                const uint32_t hi = (w << 5) + 32 > s ? s - (w << 5) : 32u;   // clear bits [lo, hi) of word w
                p.marks[w] &= ~((hi == 32 ? 0xFFFFFFFFu : (1u << hi) - 1u) & ~((1u << lo) - 1u));
            }
            syncwarp();
            s = piece = q + 1;
            continue;
        }
        if (kMeet && any(mine && ((p.marks[(s + lane) >> 5] >> ((s + lane) & 31u)) & 1u))) return K8_MET;
        if (kMark && lane == 0) {
            // segments start at multiples of 32 and only starts below the segment end are marked, so every word
            // written with a non-zero value belongs to this warp's segment alone
            p.marks[s >> 5] |= inm << (s & 31u);
            const uint32_t hi = (s & 31u) ? inm >> (32 - (s & 31u)) : 0u;
            if (hi) p.marks[(s >> 5) + 1] |= hi;
        }
        const uint32_t olen = mine ? (uint32_t)len : 0u;
        uint32_t incl = olen;
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
            const uint32_t t = shfl_up(incl, k);
            if (lane >= (unsigned)k) incl += t;
        }
        if (kCut) {
            const uint64_t D = obase + d + (incl - olen);
            if (mine && D < dn && (D & 0xFFFFu) == 0) p.cut[D >> 16] = s + lane;
            if (any(mine && (D & 0xFFFFu) + olen > 65536u)) return K8_BAD;
        }
        d += shfl(incl, 31);
        s += shfl((uint32_t)end, 31 - clz(inm));
    }
    *out = d;
    return s;
}

SB_DEVICE void k8_header_body(const RawPlan& p) {
    if (thread_idx() != 0 || block_idx() != 0) return;
    RawCtl c;
    uint64_t v = 0;
    const uint32_t hl = p.n ? k2_read_header(p.in, (uint32_t)p.n, &v) : 0;
    c.decline = (hl == 0 || v > kMaxInput || v > p.cap) ? 1u : 0u;
    c.dn = c.decline ? 0 : v; c.hl = hl; c.nblk = (uint32_t)((c.dn + 65535) >> 16); c.out_len = 0;
    *p.ctl = c;
}

// The per-segment steps below take segment k (< p.nseg) of a stream that is not declined (k8_cuts_seg checks that
// itself). The single-stream kernels give one warp per segment of p; the batch kernels (k8b_*) one warp per segment of
// any unit's view.
SB_DEVICE void k8_chains_seg(const RawPlan& p, uint64_t k) {
    const uint64_t b = k * p.seg, lim = b + p.seg < p.n ? b + p.seg : p.n;
    const uint64_t start = k ? b : p.ctl->hl;
    uint64_t out;
    const uint64_t x = start < lim ? k8_walk<true, false>(p, start, lim, 0, 0, &out) : start;
    if (lane_id() == 0) p.X[k] = x;
}
SB_DEVICE void k8_chains_body(const RawPlan& p) {
    const uint64_t k = (uint64_t)block_idx() * (block_dim() >> 5) + warp_id();
    if (k >= p.nseg || k8_declined(p)) return;
    k8_chains_seg(p, k);
}

SB_DEVICE void k8_merge_seg(const RawPlan& p, uint64_t k) {                  // k >= 1
    const uint64_t e = p.X[k - 1], lim = (k + 1) * p.seg < p.n ? (k + 1) * p.seg : p.n;
    uint64_t out;
    const uint64_t x = e < lim ? k8_walk<false, false, true>(p, e, lim, 0, 0, &out) : e;
    if (lane_id() == 0) p.Y[k] = x == K8_MET ? p.X[k] : x;
}
SB_DEVICE void k8_merge_body(const RawPlan& p) {
    const uint64_t k = (uint64_t)block_idx() * (block_dim() >> 5) + warp_id();
    if (k == 0 || k >= p.nseg || k8_declined(p)) return;
    k8_merge_seg(p, k);
}

SB_DEVICE void k8_stitch_body(const RawPlan& p) {
    const unsigned T = K8_STITCH_THREADS, t = thread_idx();
    uint64_t* sX = (uint64_t*)smem();                                // X_{k-1}, Y_k of one tile of segments
    uint64_t* sY = sX + T;
    uint32_t* sOk = (uint32_t*)(sY + T);
    uint64_t e = p.ctl->hl;                                          // thread 0's chain state
    if (t == 0) sOk[0] = !p.ctl->decline;
    syncthreads();
    for (uint64_t k0 = 0; k0 < p.nseg && sOk[0]; k0 += T) {
        const uint64_t k = k0 + t;
        if (k < p.nseg && k) { sX[t] = p.X[k - 1]; sY[t] = p.Y[k]; }
        syncthreads();
        if (t == 0) {
            bool ok = true;
            for (uint32_t j = 0; j < T && k0 + j < p.nseg && ok; j++) {
                const uint64_t k1 = k0 + j;
                p.ent[k1] = e;
                // segment 0 is walked from the header end too: its canonical parse is the true one unless it was
                // restarted, and then the walk meets the element that made it restart
                const uint64_t x = (k1 != 0 && e == sX[j]) ? sY[j] : k8_resolve(p, k1, e);
                p.ext[k1] = x;
                ok = x != K8_BAD;
                e = x;
            }
            sOk[0] = ok;
        }
        syncthreads();
    }
    if (t == 0 && (!sOk[0] || e != p.n)) p.ctl->decline = 1;
}

SB_DEVICE void k8_counts_seg(const RawPlan& p, uint64_t k) {
    const uint64_t e = p.ent[k], x = p.ext[k];
    uint64_t out = 0;
    if (e < x) k8_walk<false, false>(p, e, x, 0, 0, &out);
    if (lane_id() == 0) p.cnt[k] = (uint32_t)out;
}
SB_DEVICE void k8_counts_body(const RawPlan& p) {
    const uint64_t k = (uint64_t)block_idx() * (block_dim() >> 5) + warp_id();
    if (k >= p.nseg || k8_declined(p)) return;
    k8_counts_seg(p, k);
}
SB_DEVICE void k8_scan_local_body(const RawPlan& p) {
    const uint32_t* cnt = p.cnt;
    const bool live = !p.ctl->decline;
    scan_local_body(p.nseg, [&](uint32_t i) { return live ? cnt[i] : 0u; }, p.offs, p.tiles);
}
SB_DEVICE void k8_scan_tiles_body(const RawPlan& p) { scan_tiles_body(p.nseg, 0, p.tiles); }

// total(): output bytes of the stream's segments (checked against dn by segment 0); obase(): output position of the
// element at ent[k]. Both are evaluated only where they are needed.
template <class Total, class Obase>
SB_DEVICE void k8_cuts_seg(const RawPlan& p, uint64_t k, Total total, Obase obase) {
    RawCtl* ctl = p.ctl;
    if (k8_declined(p)) return;
    const uint64_t dn = ctl->dn;
    if (k == 0 && lane_id() == 0) {
        if (total() != dn) ctl->decline = 1;
        p.cut[ctl->nblk] = (uint32_t)p.n;
    }
    const uint64_t e = p.ent[k], x = p.ext[k];
    uint64_t out;
    if (e < x && k8_walk<false, true>(p, e, x, obase(), dn, &out) == K8_BAD && lane_id() == 0)
        ctl->decline = 1;
}
SB_DEVICE void k8_cuts_body(const RawPlan& p) {
    const uint64_t k = (uint64_t)block_idx() * (block_dim() >> 5) + warp_id();
    if (k >= p.nseg) return;
    k8_cuts_seg(p, k, [&] { return p.tiles[(p.nseg + K4_TILE - 1) / K4_TILE]; },
                [&] { return p.tiles[k / K4_TILE] + p.offs[k]; });
}

// block j of a split stream (dn: its decompressed length), decoded alone by the calling warp
SB_DEVICE void k8_block(const RawPlan& p, uint64_t j, uint64_t dn, uint32_t* elems) {
    const uint32_t a = p.cut[j], b = p.cut[j + 1];
    const uint64_t want = dn - (j << 16) < 65536 ? dn - (j << 16) : 65536;
    const uint32_t code = k2_decode_stream<false>(p.in + a, b - a, p.out + (j << 16), want, nullptr, nullptr, elems);
    if (code != SB_OK && lane_id() == 0) p.ctl->decline = 1;
}
SB_DEVICE void k8_blocks_body(const RawPlan& p) {
    RawCtl* ctl = p.ctl;
    if (k8_declined(p)) return;
    uint32_t* elems = (uint32_t*)smem() + warp_id() * 64;
    const uint32_t nblk = ctl->nblk;
    const uint64_t dn = ctl->dn;
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t j = (uint64_t)block_idx() * wpb + warp_id(); j < nblk; j += nwarps) k8_block(p, j, dn, elems);
}

SB_DEVICE void k8_fallback_body(const RawPlan& p) {
    RawCtl* ctl = p.ctl;
    sb_frame_result* r = p.result;
    if (!k8_declined(p)) {
        if (lane_id() == 0) {
            r->status.code = SB_OK; r->status._pad = 0; r->status.a = r->status.b = r->status.c = 0;
            r->bytes = ctl->dn; r->nchunks = ctl->nblk; r->_pad = 0;
        }
        return;
    }
    const uint32_t code = k2_decode_stream(p.in, (uint32_t)p.n, p.out, p.cap, &r->status, &ctl->out_len, (uint32_t*)smem());
    syncwarp();
    if (lane_id() == 0) { r->bytes = code == SB_OK ? ctl->out_len : 0; r->nchunks = 0; r->_pad = 0; }
}


// ---------------------------------------------------------------------------------------------------------- K8 batch
// K8 over a batch of raw streams (sb_decompress_batch_device_ws). Every unit whose header announces more than 65,536
// bytes is split and its blocks decoded as above; the per-segment steps run on an ordinary RawPlan *view* of the unit
// (its own input, output, control record and slices of the shared arrays), so the batch adds only the unit dimension.
//   k8b_plan        thread per unit: the split verdict (RawCtl per unit) and three per-unit counts -- segments, blocks,
//                   mark words -- scanned by K4's two-level scan (k8b_plan_tiles finishes it); Σ in_lens -> bctl.
//   k8b_chains, k8b_merge, k8b_counts, k8b_cuts   warp per segment of the global segment list: binary search for
//                   (unit, local segment), then the single-stream step on the unit's view.
//   k8b_stitch      CTA per split unit: k8_stitch_body on its view.
//   k8b_scan_*      K4's scan over the global segment list's output counts; a segment's output base is the scan
//                   value minus the value at its unit's first segment.
//   k8b_blocks      warp per block of the global block list.
//   k8b_finish      warp per unit, always: split units get Ok, dn and their block count; every other unit (never split,
//                   or declined anywhere above) is decoded by k2_decode_stream exactly as k2_decompress_body does.
// A unit is split only when it has more than one block, fits its output, and its header announces no more output than
// its body can encode (64 bytes per 3-byte copy-2 is the densest element). That bounds the blocks by the compressed
// bytes, so every slice is sized from the caller's bound `in_bytes` on Σ in_lens; when the lengths on the device sum
// to more than that, nothing is split and every unit takes the one-warp path.
static const uint64_t K8B_MAX_IN_BYTES = 1ull << 36;   // larger bounds are clamped: 2^36 / 32 mark words per tile fit u32
static const uint32_t K8B_MAX_COUNT = 1u << 31;

struct RawBatchCtl { unsigned long long in_total; };    // Σ in_lens (zeroed before k8b_plan)

struct RawBatchPlan {
    sb_batch b;                        // the units (device descriptors)
    uint64_t in_bytes;                 // the caller's bound on Σ in_lens (clamped to K8B_MAX_IN_BYTES)
    uint64_t seg;                      // segment length, as for one stream
    uint32_t* unit_blocks;             // optional: blocks decoded in parallel per unit, 0 for the one-warp path
    RawBatchCtl* bctl;
    RawCtl* uctl;                      // count: each unit's control record
    uint64_t *sg_offs, *sg_tiles;      // scan over units (count + 1 entries) of their segments,
    uint64_t *bk_offs, *bk_tiles;      // ... blocks,
    uint64_t *wd_offs, *wd_tiles;      // ... mark words
    uint32_t* marks;                   // per-unit slices, zeroed by each segment's k8b_chains warp
    uint64_t *X, *Y, *ent, *ext;       // global segment list
    uint32_t* cnt;
    uint64_t *offs, *tiles;            // scan of cnt over nseg_cap + 1 entries
    uint32_t nseg_cap;                 // segments the scratch holds
    uint32_t* cut;                     // unit i: its blocks' prefix + i, nblk + 1 entries
};

// Scratch layout (host side): every array 256-byte aligned from `scratch` (null: just the size). Returns the bytes used.
inline uint64_t k8b_carve(void* scratch, uint32_t count, uint64_t in_bytes, RawBatchPlan* q) {
    const uint64_t in = in_bytes < K8B_MAX_IN_BYTES ? in_bytes : K8B_MAX_IN_BYTES;
    const uint64_t units = (uint64_t)count + 1;
    const uint64_t segs = in / K8_SEG_MIN + count;                      // Σ ceil(n_i / seg)
    const uint64_t words = in / 32 + 2 * (uint64_t)count;               // Σ (n_i >> 5) + 2
    const uint64_t cuts = in / 3072 + 2 * (uint64_t)count + 1;          // Σ ceil(dn_i / 65536) + 1, dn_i <= n_i * 64 / 3
    const uintptr_t base = ((uintptr_t)scratch + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    RawBatchPlan p;
    p.in_bytes = in;
    p.nseg_cap = (uint32_t)segs;
    p.bctl = (RawBatchCtl*)take(sizeof(RawBatchCtl));
    p.uctl = (RawCtl*)take(count * sizeof(RawCtl));
    uint64_t** scans[3][2] = {{&p.sg_offs, &p.sg_tiles}, {&p.bk_offs, &p.bk_tiles}, {&p.wd_offs, &p.wd_tiles}};
    for (auto& sc : scans) { *sc[0] = (uint64_t*)take((units + 1) * 8); *sc[1] = (uint64_t*)take((units / K4_TILE + 3) * 8); }
    p.marks = (uint32_t*)take(words * 4);
    p.X = (uint64_t*)take((segs + 1) * 8);
    p.Y = (uint64_t*)take((segs + 1) * 8);
    p.ent = (uint64_t*)take((segs + 1) * 8);
    p.ext = (uint64_t*)take((segs + 1) * 8);
    p.cnt = (uint32_t*)take((segs + 1) * 4);
    p.offs = (uint64_t*)take((segs + 2) * 8);
    p.tiles = (uint64_t*)take(((segs + 1) / K4_TILE + 3) * 8);
    p.cut = (uint32_t*)take(cuts * 4);
    if (q) {
        p.b = q->b; p.seg = q->seg; p.unit_blocks = q->unit_blocks;
        *q = p;
    }
    return at + 256;
}

// exclusive prefix at i of a two-level scan
SB_DEVICE uint64_t k8b_at(const uint64_t* offs, const uint64_t* tiles, uint64_t i) { return tiles[i / K4_TILE] + offs[i]; }
// Σ in_lens over the bound: nothing is split
SB_DEVICE bool k8b_over(const RawBatchPlan& q) { return q.bctl->in_total > q.in_bytes; }
// the unit whose slice of a per-unit scan holds global index g < S(count): the last u with S(u) <= g
SB_DEVICE uint32_t k8b_unit_of(const uint64_t* offs, const uint64_t* tiles, uint32_t count, uint64_t g) {
    uint32_t lo = 0, hi = count;                                     // S(lo) <= g < S(hi)
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (k8b_at(offs, tiles, mid) <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// unit u as one stream: its buffers, control record and slices (offs/tiles are the batch's global scan)
SB_DEVICE RawPlan k8b_view(const RawBatchPlan& q, uint32_t u) {
    RawPlan p;
    p.in = unit_in(q.b, u); p.n = unit_in_len(q.b, u);
    p.out = unit_out(q.b, u); p.cap = unit_out_cap(q.b, u);
    p.result = nullptr;
    p.seg = q.seg; p.nseg = (uint32_t)((p.n + q.seg - 1) / q.seg);
    p.ctl = q.uctl + u;
    const uint64_t s0 = k8b_at(q.sg_offs, q.sg_tiles, u);
    p.marks = q.marks + k8b_at(q.wd_offs, q.wd_tiles, u);
    p.X = q.X + s0; p.Y = q.Y + s0; p.ent = q.ent + s0; p.ext = q.ext + s0; p.cnt = q.cnt + s0;
    p.offs = q.offs; p.tiles = q.tiles;
    p.cut = q.cut + k8b_at(q.bk_offs, q.bk_tiles, u) + u;
    return p;
}

SB_DEVICE void k8b_plan_body(const RawBatchPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t ns = 0, nb = 0, nw = 0;
    uint64_t n = 0;
    if (i < count) {
        n = unit_in_len(q.b, (uint32_t)i);
        const uint64_t cap = unit_out_cap(q.b, (uint32_t)i);
        uint64_t v = 0;
        const uint32_t hl = n ? k2_read_header(unit_in(q.b, (uint32_t)i), (uint32_t)n, &v) : 0;
        const bool split = hl && v > kMaxBlock && v <= kMaxInput && v <= cap && v * 3 <= (n - hl) * 64;
        RawCtl c;
        c.decline = split ? 0u : 1u; c.dn = split ? v : 0; c.hl = hl; c.nblk = (uint32_t)((c.dn + 65535) >> 16); c.out_len = 0;
        q.uctl[i] = c;
        if (split) { ns = (uint32_t)((n + q.seg - 1) / q.seg); nb = c.nblk; nw = (uint32_t)((n >> 5) + 2); }
    }
    uint64_t t = n;
#pragma unroll
    for (unsigned m = 16; m; m >>= 1) t += shfl(t, lane_id() ^ m);
    if (lane_id() == 0 && t) atomic_add(&q.bctl->in_total, (unsigned long long)t);
    scan_local_body(count + 1, [&](uint32_t) { return ns; }, q.sg_offs, q.sg_tiles);
    syncthreads();
    scan_local_body(count + 1, [&](uint32_t) { return nb; }, q.bk_offs, q.bk_tiles);
    syncthreads();
    scan_local_body(count + 1, [&](uint32_t) { return nw; }, q.wd_offs, q.wd_tiles);
}
SB_DEVICE void k8b_plan_tiles_body(const RawBatchPlan& q) {
    scan_tiles_body(q.b.count + 1, 0, q.sg_tiles);
    syncthreads();
    scan_tiles_body(q.b.count + 1, 0, q.bk_tiles);
    syncthreads();
    scan_tiles_body(q.b.count + 1, 0, q.wd_tiles);
}

// f(view, local segment k, global segment g) for every segment of the global list, one warp each
template <class F>
SB_DEVICE void k8b_segments(const RawBatchPlan& q, F f) {
    if (k8b_over(q)) return;
    const uint32_t count = q.b.count;
    const uint64_t total = k8b_at(q.sg_offs, q.sg_tiles, count);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t g = (uint64_t)block_idx() * wpb + warp_id(); g < total; g += nwarps) {
        const RawPlan p = k8b_view(q, k8b_unit_of(q.sg_offs, q.sg_tiles, count, g));
        f(p, g - (uint64_t)(p.X - q.X), g);
    }
}

SB_DEVICE void k8b_chains_body(const RawBatchPlan& q) {
    k8b_segments(q, [&](const RawPlan& p, uint64_t k, uint64_t) {
        if (k8_declined(p)) return;
        // the segment's own words of the unit's mark slice (k8_walk marks and clears no others)
        const uint32_t w0 = (uint32_t)(k * (p.seg >> 5));
        const uint32_t w1 = (uint32_t)(k + 1 == p.nseg ? (p.n >> 5) + 2 : (k + 1) * (p.seg >> 5));
        for (uint32_t w = w0 + lane_id(); w < w1; w += 32) p.marks[w] = 0;
        syncwarp();
        k8_chains_seg(p, k);
    });
}
SB_DEVICE void k8b_merge_body(const RawBatchPlan& q) {
    k8b_segments(q, [&](const RawPlan& p, uint64_t k, uint64_t) {
        if (k != 0 && !k8_declined(p)) k8_merge_seg(p, k);
    });
}
SB_DEVICE void k8b_stitch_body(const RawBatchPlan& q) {
    if (k8b_over(q)) return;
    for (uint32_t u = block_idx(); u < q.b.count; u += grid_dim()) {
        if (q.uctl[u].decline) continue;                             // the same for every thread: only this CTA writes it
        k8_stitch_body(k8b_view(q, u));
        syncthreads();
    }
}
SB_DEVICE void k8b_counts_body(const RawBatchPlan& q) {
    k8b_segments(q, [&](const RawPlan& p, uint64_t k, uint64_t g) {
        if (!k8_declined(p)) k8_counts_seg(p, k);
        else if (lane_id() == 0) q.cnt[g] = 0;                       // scanned with the rest
    });
}
SB_DEVICE void k8b_scan_local_body(const RawBatchPlan& q) {
    const uint64_t total = k8b_over(q) ? 0 : k8b_at(q.sg_offs, q.sg_tiles, q.b.count);
    const uint32_t* cnt = q.cnt;
    scan_local_body(q.nseg_cap + 1, [&](uint32_t g) { return g < total ? cnt[g] : 0u; }, q.offs, q.tiles);
}
SB_DEVICE void k8b_scan_tiles_body(const RawBatchPlan& q) { scan_tiles_body(q.nseg_cap + 1, 0, q.tiles); }
SB_DEVICE void k8b_cuts_body(const RawBatchPlan& q) {
    k8b_segments(q, [&](const RawPlan& p, uint64_t k, uint64_t g) {
        if (k8_declined(p)) return;
        // Unit-relative positions are exact modulo 2^32 (the scan's tiles may mix units and wrap), and a split unit's
        // output is below 2^32. A segment whose elements run past dn declines: it exists whenever the unit's true
        // total exceeds dn, and its own base is below 2^32, so a total that wrapped cannot pass for dn.
        const uint64_t s0 = g - k, first = k8b_at(q.offs, q.tiles, s0);
        const uint64_t obase = (uint32_t)(k8b_at(q.offs, q.tiles, g) - first);
        if (lane_id() == 0 && obase + p.cnt[k] > p.ctl->dn) p.ctl->decline = 1;
        k8_cuts_seg(p, k, [&] { return (uint64_t)(uint32_t)(k8b_at(q.offs, q.tiles, s0 + p.nseg) - first); },
                    [&] { return obase; });
    });
}
SB_DEVICE void k8b_blocks_body(const RawBatchPlan& q) {
    if (k8b_over(q)) return;
    uint32_t* elems = (uint32_t*)smem() + warp_id() * 64;
    const uint32_t count = q.b.count;
    const uint64_t total = k8b_at(q.bk_offs, q.bk_tiles, count);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t g = (uint64_t)block_idx() * wpb + warp_id(); g < total; g += nwarps) {
        const uint32_t u = k8b_unit_of(q.bk_offs, q.bk_tiles, count, g);
        const RawPlan p = k8b_view(q, u);
        if (k8_declined(p)) continue;
        const uint64_t j = g - (uint64_t)(p.cut - q.cut - u);
        if (p.cut[j] > p.cut[j + 1] || p.cut[j + 1] > p.n) {         // cannot happen once the cuts were accepted
            if (lane_id() == 0) p.ctl->decline = 1;
            continue;
        }
        k8_block(p, j, p.ctl->dn, elems);
    }
}
SB_DEVICE void k8b_finish_body(const RawBatchPlan& q) {
    const BatchDesc& b = q.b;
    const bool over = k8b_over(q);
    const unsigned wpb = block_dim() >> 5;
    uint32_t* elems = (uint32_t*)smem() + warp_id() * 64;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t u = (uint64_t)block_idx() * wpb + warp_id(); u < b.count; u += nwarps) {
        const uint32_t i = (uint32_t)u;
        const RawCtl& c = q.uctl[i];
        if (!over && !c.decline) {
            if (lane_id() == 0) {
                if (b.statuses) set_status(&b.statuses[i], SB_OK, 0, 0, 0);
                if (b.out_lens) b.out_lens[i] = (uint32_t)c.dn;
                if (q.unit_blocks) q.unit_blocks[i] = c.nblk;
            }
            continue;
        }
        if (lane_id() == 0) {
            if (b.out_lens) b.out_lens[i] = 0;
            if (q.unit_blocks) q.unit_blocks[i] = 0;
        }
        k2_decode_stream(unit_in(b, i), unit_in_len(b, i), unit_out(b, i), unit_out_cap(b, i),
                         b.statuses ? &b.statuses[i] : nullptr, b.out_lens ? &b.out_lens[i] : nullptr, elems);
    }
}

}  // namespace sbk

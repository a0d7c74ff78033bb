// k9_raw_batch_compress.cuh -- K9: raw compress of a batch of units of any length (sb_compress_batch_device_ws).
//
// Replaces, per unit, reference src/compress.rs:99-154 (Encoder::compress: the two length checks, the varint header
// and the 64 KB block loop). Blocks are independent by format (the reference resets its table for every block,
// :129-152), so every unit is cut into its blocks and all blocks of the batch go through ONE K1 launch, unchanged:
//   k9_plan        thread per unit: the reference's checks and the unit's class (rejected, empty, one block, more than
//                  one block); Σ n over multi-block units -> ctl.
//   k9_scan_*      K4's two-level scan of every unit's slot count (its blocks when it has more than one, else 0).
//   k9_fill        thread per K1 entry. Entry u < count is unit u's single block, compressed straight into the
//                  caller's output behind the unit's header (a batch of <= 64 KB units pays no copy); entry count + g
//                  is slot g of the global slot list (binary search for its unit). Entries past the device-side total
//                  get length 0, which K1 finishes in two barriers: the grid is sized from the host's bound.
//   K1             flags 0 (no per-block header), slots of kSlotStride.
//   k9_bscan_*     the same scan over the slots' compressed lengths; a block's offset inside its unit is its scan
//                  value minus the value at its unit's first slot.
//   k9_gather      warp per slot: the block body to out_i + hl_i + offset.
//   k9_finish      thread per unit, always: the varint header, out_lens and the status.
// Only units over 64 KB use slots, so the scratch is sized from the caller's bound `in_bytes` on their Σ n: a unit of
// n > 65536 bytes takes ceil(n / 65536) <= floor(n / 65536) + 1 slots, so Σ <= floor(in_bytes / 65536) + min(count,
// floor(in_bytes / 65537)). When the lengths on the device sum to more than that, no unit gets slots and every
// multi-block unit is SB_E_INVALID{sum, in_bytes}.
#pragma once
#include "k1_compress.cuh"
#include "k4_frame.cuh"
#include "k8_raw_split.cuh"

namespace sbk {

static const uint32_t K9_MAX_COUNT = 1u << 31;

enum : uint32_t { K9_TOO_BIG = 0, K9_TOO_SMALL = 1, K9_EMPTY = 2, K9_SINGLE = 3, K9_MULTI = 4 };

struct RawCompressCtl { unsigned long long in_total; };   // Σ n over multi-block units (zeroed before k9_plan)

struct RawCompressPlan {
    sb_batch b;                        // the units (device descriptors)
    uint64_t in_bytes;                 // the caller's bound on Σ n over units of more than 65,536 bytes
    uint32_t nslot;                    // slots the scratch holds
    uint32_t nk;                       // K1 entries: count + nslot
    RawCompressCtl* ctl;
    uint32_t* cls;                     // count: K9_* class of every unit
    uint64_t *sl_offs, *sl_tiles;      // scan over units (count + 1 entries) of their slot counts
    const uint8_t** k1_in;             // nk: K1's unit descriptors
    uint8_t** k1_out;
    uint32_t *k1_lens, *k1_clens;
    uint64_t *bo_offs, *bo_tiles;      // scan over slots (nslot + 1 entries) of their compressed lengths
    uint8_t* slots;                    // nslot x kSlotStride
};

// slots the scratch needs for a bound in_bytes on Σ n over multi-block units
inline uint64_t k9_slot_bound(uint32_t count, uint64_t in_bytes) {
    const uint64_t units = in_bytes / (kMaxBlock + 1);
    return in_bytes / kMaxBlock + (units < count ? units : count);
}

// Scratch layout (host side): every array 256-byte aligned from `scratch` (null: just the size). Returns the bytes used,
// or UINT64_MAX when count + slots does not fit a K1 launch (a u32 entry count, plus one for the scans).
inline uint64_t k9_carve(void* scratch, uint32_t count, uint64_t in_bytes, RawCompressPlan* q) {
    const uint64_t nslot = k9_slot_bound(count, in_bytes);
    const uint64_t nk = (uint64_t)count + nslot;
    if (nk >= 0xFFFFFFFFull) return ~0ull;
    const uintptr_t base = ((uintptr_t)scratch + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    RawCompressPlan p;
    p.nslot = (uint32_t)nslot; p.nk = (uint32_t)nk;
    p.ctl = (RawCompressCtl*)take(sizeof(RawCompressCtl));
    p.cls = (uint32_t*)take((uint64_t)count * 4);
    p.sl_offs = (uint64_t*)take(((uint64_t)count + 2) * 8);
    p.sl_tiles = (uint64_t*)take(((uint64_t)count + 1) / K4_TILE * 8 + 24);
    p.k1_in = (const uint8_t**)take(nk * 8);
    p.k1_out = (uint8_t**)take(nk * 8);
    p.k1_lens = (uint32_t*)take(nk * 4);
    p.k1_clens = (uint32_t*)take(nk * 4);
    p.bo_offs = (uint64_t*)take((nslot + 2) * 8);
    p.bo_tiles = (uint64_t*)take((nslot + 1) / K4_TILE * 8 + 24);
    p.slots = (uint8_t*)take(nslot * kSlotStride);
    if (q) {
        p.b = q->b; p.in_bytes = in_bytes;
        *q = p;
    }
    return at + 256;
}

// max_compress_len(n) without its 0 for "too big" (src/compress.rs:42-53)
SB_DEVICE uint64_t k9_need(uint64_t n) { return 32 + n + n / 6; }
SB_DEVICE uint32_t k9_varint_len(uint64_t n) { uint32_t k = 1; while (n >= 0x80) { n >>= 7; k++; } return k; }
SB_DEVICE bool k9_over(const RawCompressPlan& q) { return q.ctl->in_total > q.in_bytes; }
// slots of unit u: its blocks when it has more than one and the batch is within its bound
SB_DEVICE uint32_t k9_slots(const RawCompressPlan& q, uint32_t u) {
    if (q.cls[u] != K9_MULTI || k9_over(q)) return 0;
    return (uint32_t)(((uint64_t)unit_in_len(q.b, u) + kMaxBlock - 1) / kMaxBlock);
}

SB_DEVICE void k9_plan_body(const RawCompressPlan& q) {
    const uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx();
    uint64_t multi = 0;
    if (i < q.b.count) {
        const uint64_t n = unit_in_len(q.b, (uint32_t)i), cap = unit_out_cap(q.b, (uint32_t)i);
        uint32_t c;
        if (k9_need(n) > kMaxInput) c = K9_TOO_BIG;                     // (:104-109)
        else if (cap < k9_need(n)) c = K9_TOO_SMALL;                   // (:110-115)
        else if (n == 0) c = K9_EMPTY;
        else if (n <= kMaxBlock) c = K9_SINGLE;
        else { c = K9_MULTI; multi = n; }
        q.cls[i] = c;
    }
#pragma unroll
    for (unsigned m = 16; m; m >>= 1) multi += shfl(multi, lane_id() ^ m);
    if (lane_id() == 0 && multi) atomic_add(&q.ctl->in_total, (unsigned long long)multi);
}
SB_DEVICE void k9_scan_local_body(const RawCompressPlan& q) {
    const uint32_t count = q.b.count;
    scan_local_body(count + 1, [&](uint32_t u) { return u < count ? k9_slots(q, u) : 0u; }, q.sl_offs, q.sl_tiles);
}
SB_DEVICE void k9_scan_tiles_body(const RawCompressPlan& q) { scan_tiles_body(q.b.count + 1, 0, q.sl_tiles); }

SB_DEVICE void k9_fill_body(const RawCompressPlan& q) {
    const uint64_t e = (uint64_t)block_idx() * block_dim() + thread_idx();
    if (e >= q.nk) return;
    const uint32_t count = q.b.count;
    const uint8_t* in = nullptr;
    uint8_t* out = nullptr;
    uint32_t len = 0;
    if (e < count) {
        const uint32_t u = (uint32_t)e;
        if (q.cls[u] == K9_SINGLE) {
            len = unit_in_len(q.b, u);
            in = unit_in(q.b, u);
            out = unit_out(q.b, u) + k9_varint_len(len);
        }
    } else {
        const uint64_t g = e - count;
        if (g < k8b_at(q.sl_offs, q.sl_tiles, count)) {
            const uint32_t u = k8b_unit_of(q.sl_offs, q.sl_tiles, count, g);
            const uint64_t j = g - k8b_at(q.sl_offs, q.sl_tiles, u), n = unit_in_len(q.b, u);
            const uint64_t left = n - j * kMaxBlock;
            len = left > kMaxBlock ? kMaxBlock : (uint32_t)left;
            in = unit_in(q.b, u) + j * kMaxBlock;
            out = q.slots + g * kSlotStride;
        }
    }
    q.k1_in[e] = in; q.k1_out[e] = out; q.k1_lens[e] = len;
}

// K1's batch over the entries. The uniform cap is only K1's check that a slot holds max_compress_len(block): a block
// compressed in place fits the caller's buffer behind the header, which holds max_compress_len(n) bytes.
inline sb_batch k9_k1_batch(const RawCompressPlan& q) {
    sb_batch k;
    memset(&k, 0, sizeof k);
    k.in_ptrs = q.k1_in; k.in_lens = q.k1_lens;
    k.out_ptrs = q.k1_out; k.out_cap_uniform = kSlotStride;
    k.out_lens = q.k1_clens; k.count = q.nk;
    return k;
}

SB_DEVICE void k9_bscan_local_body(const RawCompressPlan& q) {
    const uint32_t* clens = q.k1_clens + q.b.count;
    const uint32_t nslot = q.nslot;
    scan_local_body(nslot + 1, [&](uint32_t g) { return g < nslot ? clens[g] : 0u; }, q.bo_offs, q.bo_tiles);
}
SB_DEVICE void k9_bscan_tiles_body(const RawCompressPlan& q) { scan_tiles_body(q.nslot + 1, 0, q.bo_tiles); }

SB_DEVICE void k9_gather_body(const RawCompressPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t total = k8b_at(q.sl_offs, q.sl_tiles, count);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t g = (uint64_t)block_idx() * wpb + warp_id(); g < total; g += nwarps) {
        const uint32_t u = k8b_unit_of(q.sl_offs, q.sl_tiles, count, g);
        const uint64_t first = k8b_at(q.sl_offs, q.sl_tiles, u);
        const uint64_t off = k8b_at(q.bo_offs, q.bo_tiles, g) - k8b_at(q.bo_offs, q.bo_tiles, first);
        uint8_t* dst = unit_out(q.b, u) + k9_varint_len(unit_in_len(q.b, u)) + off;
        warp_copy_t<true>(dst, q.slots + g * kSlotStride, q.k1_clens[count + g]);
    }
}

SB_DEVICE void k9_finish_body(const RawCompressPlan& q) {
    const BatchDesc& b = q.b;
    const uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx();
    if (i >= b.count) return;
    const uint32_t u = (uint32_t)i, c = q.cls[u];
    const uint64_t n = unit_in_len(b, u);
    sb_error* st = b.statuses ? &b.statuses[u] : nullptr;
    if (c == K9_TOO_BIG) { b.out_lens[u] = 0; set_status(st, SB_TOO_BIG, n, kMaxInput, 0); return; }
    if (c == K9_TOO_SMALL) { b.out_lens[u] = 0; set_status(st, SB_BUFFER_TOO_SMALL, unit_out_cap(b, u), k9_need(n), 0); return; }
    if (c == K9_MULTI && k9_over(q)) { b.out_lens[u] = 0; set_status(st, SB_E_INVALID, q.ctl->in_total, q.in_bytes, 0); return; }
    uint64_t body = 0;
    if (c == K9_SINGLE) body = q.k1_clens[u];
    else if (c == K9_MULTI) {
        const uint64_t s0 = k8b_at(q.sl_offs, q.sl_tiles, u), s1 = k8b_at(q.sl_offs, q.sl_tiles, u + 1);
        body = k8b_at(q.bo_offs, q.bo_tiles, s1) - k8b_at(q.bo_offs, q.bo_tiles, s0);
    }
    uint8_t* out = unit_out(b, u);
    uint32_t hl = 0;                                                     // varint header (src/bytes.rs:61-70)
    uint64_t v = n;
    while (v >= 0x80) { out[hl++] = (uint8_t)v | 0x80; v >>= 7; }
    out[hl++] = (uint8_t)v;
    b.out_lens[u] = (uint32_t)(hl + body);
    set_status(st, SB_OK, 0, 0, 0);
}

}  // namespace sbk

// k19_validate.cuh -- K19: frame validation of a batch of streams (sb_frame_validate_batch_device_ws).
//
// Gives every unit exactly the status, out_lens and d_unit_chunks of sb_frame_decode_batch_device_ws with every cap
// 2^32 - 1, without writing a decoded byte outside the scratch. K11's sequence runs unchanged up to k11_oscan_* on a copy
// of the batch without output pointers and with caps of 2^32 - 1; k11_decode is replaced by
//   k19_validate    warp w owns staging slot w of a pool of min(max_chunks, 4,096) slots of 64 KiB (K15's policy: at
//                   most 256 MiB) and takes the chunk table's slots one at a time from a counter; it skips those that
//                   hold no live chunk of a unit that fits. A compressed chunk is decoded into the warp's slot and
//                   checksummed there; a stored chunk is checksummed in place in the input. The first failing chunk per
//                   unit by atomic_min, as k11_decode does. Every warp of the pool is resident at once, so a fixed
//                   stride (j = w, w + 4,096, ...) would leave the kernel waiting on the warps whose chunks happened to
//                   be slowest; the counter hands the next chunk to whichever warp is free (DESIGN.md section 5).
// and k11_finish then writes the results unchanged. Every decision is K5's: the chunk's decode status (K2 over the same
// body with the same bounds) and its CRC over the same bytes.
#pragma once
#include "k11_frame_batch_decode.cuh"
#include "k15_raw_table.cuh"

namespace sbk {

struct FrameValidatePlan {
    FrameDecodeBatchPlan q;            // K11's plan over the copy of the batch
    uint8_t* slots;                    // nslots * 64 KiB
    uint32_t nslots;
    uint32_t* next;                    // the next chunk table slot to hand out (zeroed before k19_validate)
};

inline uint32_t k19_slots(uint32_t max_chunks) { return max_chunks < K15_SLOTS ? max_chunks : K15_SLOTS; }

// K11's carve, then the counter and the staging slots. Returns the bytes used (a pure function of count, in_bytes and
// max_chunks): K11's, plus the slots, plus 256.
inline uint64_t k19_carve(void* scratch, uint32_t count, uint64_t in_bytes, uint32_t max_chunks, FrameValidatePlan* t) {
    const uint64_t k11 = k11_carve(scratch, count, in_bytes, max_chunks, t ? &t->q : nullptr);
    const uint64_t slots = k19_slots(max_chunks);
    // K11's arrays end k11 - 256 bytes after the 256-byte aligned start of the scratch (k11_carve keeps 256 for the
    // alignment); the counter takes the next 256 bytes, the slots follow
    const uintptr_t base = ((uintptr_t)scratch + 255) / 256 * 256 + (k11 - 256);
    if (t) { t->next = (uint32_t*)base; t->slots = (uint8_t*)(base + 256); t->nslots = (uint32_t)slots; }
    return k11 + 256 + slots * kMaxBlock;
}

SB_DEVICE void k19_validate_body(const FrameValidatePlan& t) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const FrameDecodeBatchPlan& q = t.q;
    const unsigned wpb = block_dim() >> 5;
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id(), nw = (uint64_t)grid_dim() * wpb;
    const uint64_t active = nw < t.nslots ? nw : t.nslots;            // warps with a slot of their own
    if (w >= active) return;
    uint8_t* slot = t.slots + w * kMaxBlock;
    const uint32_t total = (uint32_t)k11_slots(q);                    // <= max_chunks < 2^22
    for (;;) {
        uint32_t j = 0;
        if (lane_id() == 0) j = atomic_add(t.next, 1u);
        j = shfl(j, 0);
        if (j >= total) break;
        const uint32_t u = k11_live_unit(q, j);
        if (u == K11_NONE || k11_need(q, u) > unit_out_cap(q.b, u)) continue;
        const FChunk c = q.chunks[j];
        const uint8_t* in = unit_in(q.b, u);
        uint32_t code = SB_OK;
        if (c.type == 0) code = k2_decode_stream(in + c.body_off, c.body_len, slot, c.dlen, &q.cst[j], nullptr, elems);
        else if (lane_id() == 0) k5_set(&q.cst[j], SB_OK);
        syncwarp();
        if (code == SB_OK) {
            const uint32_t got = k3_warp_crc32c_masked(tab, c.type == 0 ? slot : in + c.body_off, c.dlen);
            if (got != c.want_crc) { code = SB_CHECKSUM; if (lane_id() == 0) k5_set(&q.cst[j], SB_CHECKSUM, c.want_crc, got); }
        }
        if (code != SB_OK && lane_id() == 0) atomic_min(&q.uctl[u].first_bad, (uint32_t)(j - k11_range(q, u)));
        syncwarp();
    }
}

}  // namespace sbk

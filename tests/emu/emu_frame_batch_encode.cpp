// emu_frame_batch_encode.cpp -- TEST TOOLING ONLY. Frame encode of a batch of units of any length (the k10_* bodies of
// rust-snappy_b200/csrc/k10_frame_batch_encode.cuh and the k9 scans they share, around the K1 body in frame mode)
// compiled by g++ against the fiber warp emulator, exposed to tests/test_frame_batch_encode_emu.py through a C
// interface. Built by that test into tests/emu/_build/libemu_frame_batch_encode.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k10_frame_batch_encode.cuh"

static void plan_entry(void* a) { sbk::k10_plan_body(*(sbk::FrameBatchPlan*)a); }
static void scan_local_entry(void* a) { sbk::k9_scan_local_body(((sbk::FrameBatchPlan*)a)->r); }
static void scan_tiles_entry(void* a) { sbk::k9_scan_tiles_body(((sbk::FrameBatchPlan*)a)->r); }
static void iscan_local_entry(void* a) { sbk::k10_iscan_local_body(*(sbk::FrameBatchPlan*)a); }
static void iscan_tiles_entry(void* a) { sbk::k10_iscan_tiles_body(*(sbk::FrameBatchPlan*)a); }
static void fill_entry(void* a) { sbk::k10_fill_body(*(sbk::FrameBatchPlan*)a); }
static void bscan_local_entry(void* a) { sbk::k10_bscan_local_body(*(sbk::FrameBatchPlan*)a); }
static void bscan_tiles_entry(void* a) { sbk::k9_bscan_tiles_body(((sbk::FrameBatchPlan*)a)->r); }
static void gather_entry(void* a) { sbk::k10_gather_body(*(sbk::FrameBatchPlan*)a); }
static void finish_entry(void* a) { sbk::k10_finish_body(*(sbk::FrameBatchPlan*)a); }

struct K1Args { sb_batch b; uint64_t* rings; uint32_t* work; uint32_t* crcs; };
static void k1_entry(void* a) {
    K1Args* x = (K1Args*)a;
    sbk::k1_compress_body_multi<7, 0>(x->b, 1u, x->rings, nullptr, x->work, x->crcs);
}

extern "C" {

uint64_t emu_frame_batch_scratch_bytes(uint32_t count, uint64_t in_bytes) { return sbk::k10_carve(nullptr, count, in_bytes, nullptr); }

// sb_frame_encode_batch_device_ws under the emulator: the scratch layout of k10_carve and the launch sequence of
// launch_frame_batch in csrc/snapb200.cu, with small grids (so every grid-stride loop takes several turns) and two K1
// CTAs of 7 chains. Returns 202 (SB_E_INVALID) where the library's call-level checks fail.
int emu_frame_batch_encode(const sb_batch* b, uint64_t in_bytes, uint64_t* idx, void* scratch, uint64_t scratch_bytes) {
    if (!b || !b->out_lens || !scratch || b->count >= sbk::K9_MAX_COUNT) return 202;
    if (b->count == 0) return 0;
    const uint64_t need = sbk::k10_carve(nullptr, b->count, in_bytes, nullptr);
    if (need == ~0ull || scratch_bytes < need) return 202;
    sbk::FrameBatchPlan q;
    memset(&q, 0, sizeof q);
    q.r.b = *b; q.idx = idx;
    sbk::k10_carve(scratch, b->count, in_bytes, &q);
    memset(q.r.ctl, 0, sizeof(sbk::RawCompressCtl));
    auto blocks = [](uint64_t n, unsigned per) { return (unsigned)((n + per - 1) / per); };
    sbemu::launch(blocks(b->count, 64), 64, 0, plan_entry, &q);
    sbemu::launch(blocks((uint64_t)b->count + 1, sbk::K4_TILE), sbk::K4_TILE, 128, scan_local_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry, &q);
    if (idx) {
        sbemu::launch(blocks((uint64_t)b->count + 1, sbk::K4_TILE), sbk::K4_TILE, 128, iscan_local_entry, &q);
        sbemu::launch(1, 1024, 1024 * 8, iscan_tiles_entry, &q);
    }
    sbemu::launch(blocks(q.r.nk, 64), 64, 0, fill_entry, &q);
    std::vector<uint64_t> rings((size_t)2 * 7 * sbk::K1_RING_GW, 0xCDCDCDCDCDCDCDCDull);
    uint32_t work = 0;
    K1Args k{sbk::k9_k1_batch(q.r), rings.data(), &work, q.crcs};
    sbemu::launch(2, 7 * 64, sbk::k1_multi_smem(7, 0), k1_entry, &k);
    sbemu::launch(blocks((uint64_t)q.r.nslot + 1, sbk::K4_TILE), sbk::K4_TILE, 128, bscan_local_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, bscan_tiles_entry, &q);
    sbemu::launch(2, 64, 0, gather_entry, &q);
    sbemu::launch(2, 64, 0, finish_entry, &q);
    return 0;
}

}

// emu_encode_tables.cpp -- TEST TOOLING ONLY. Tabled batch encodes: K9's or K10's bodies around the K1 body with its
// CRC array, then the k16_* bodies of rust-snappy_b200/csrc/k16_encode_tables.cuh, compiled by g++ against the fiber warp
// emulator and exposed to tests/test_encode_tables_emu.py through a C interface. Built by that test into
// tests/emu/_build/libemu_encode_tables.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k16_encode_tables.cuh"

typedef sbk::EncodeTablesPlan T;
static void k9_plan_entry(void* a) { sbk::k9_plan_body(((T*)a)->f.r); }
static void k10_plan_entry(void* a) { sbk::k10_plan_body(((T*)a)->f); }
static void scan_local_entry(void* a) { sbk::k9_scan_local_body(((T*)a)->f.r); }
static void scan_tiles_entry(void* a) { sbk::k9_scan_tiles_body(((T*)a)->f.r); }
static void iscan_local_entry(void* a) { sbk::k10_iscan_local_body(((T*)a)->f); }
static void iscan_tiles_entry(void* a) { sbk::k10_iscan_tiles_body(((T*)a)->f); }
static void k9_fill_entry(void* a) { sbk::k9_fill_body(((T*)a)->f.r); }
static void k10_fill_entry(void* a) { sbk::k10_fill_body(((T*)a)->f); }
static void k9_bscan_local_entry(void* a) { sbk::k9_bscan_local_body(((T*)a)->f.r); }
static void k10_bscan_local_entry(void* a) { sbk::k10_bscan_local_body(((T*)a)->f); }
static void bscan_tiles_entry(void* a) { sbk::k9_bscan_tiles_body(((T*)a)->f.r); }
static void k9_gather_entry(void* a) { sbk::k9_gather_body(((T*)a)->f.r); }
static void k10_gather_entry(void* a) { sbk::k10_gather_body(((T*)a)->f); }
static void k9_finish_entry(void* a) { sbk::k9_finish_body(((T*)a)->f.r); }
static void k10_finish_entry(void* a) { sbk::k10_finish_body(((T*)a)->f); }
static void raw_size_local_entry(void* a) { sbk::k16_size_local_body<false>(*(T*)a); }
static void frame_size_local_entry(void* a) { sbk::k16_size_local_body<true>(*(T*)a); }
static void size_tiles_entry(void* a) { sbk::k16_size_tiles_body(*(T*)a); }
static void raw_export_entry(void* a) { sbk::k16_raw_export_body(*(T*)a); }
static void frame_export_entry(void* a) { sbk::k16_frame_export_body(*(T*)a); }

struct K1Args { sb_batch b; uint32_t flags; uint64_t* rings; uint32_t* work; uint32_t* crcs; };
static void k1_entry(void* a) {
    K1Args* x = (K1Args*)a;
    sbk::k1_compress_body_multi<7, 0>(x->b, x->flags, x->rings, nullptr, x->work, x->crcs);
}

extern "C" {

uint64_t emu_compress_tables_bytes(uint32_t count, uint64_t in_bytes) { return sbk::k16_raw_tables_bytes(count, in_bytes); }
uint64_t emu_frame_encode_tables_bytes(uint32_t count, uint64_t in_bytes) {
    return sbk::k16_frame_tables_bytes(count, in_bytes);
}
uint64_t emu_encode_tabled_scratch_bytes(int frame, uint32_t count, uint64_t in_bytes) {
    return frame ? sbk::k16_frame_carve(nullptr, count, in_bytes, nullptr) : sbk::k16_raw_carve(nullptr, count, in_bytes, nullptr);
}

// sb_compress_batch_tabled_device_ws (frame 0) or sb_frame_encode_batch_tabled_device_ws (frame 1) under the emulator:
// the call-level checks, the scratch layout of k16_raw_carve / k16_frame_carve and the launch sequence of
// launch_encode_tabled in csrc/snapb200.cu, with small grids (so every grid-stride loop takes several turns) and two K1
// CTAs of 7 chains. Returns 202 (SB_E_INVALID) where the library does.
int emu_encode_tabled(int frame, const sb_batch* b, uint64_t in_bytes, uint64_t* idx, void* tables, uint64_t tables_bytes,
                      uint64_t* table_offs, sb_frame_result* results, void* scratch, uint64_t scratch_bytes) {
    if (!b || !b->out_lens || !tables || !table_offs || !results || !scratch) return 202;
    if (b->count >= sbk::K9_MAX_COUNT) return 202;
    if (b->count == 0) return 0;
    const uint64_t need = emu_encode_tabled_scratch_bytes(frame, b->count, in_bytes);
    if (need == ~0ull) return 202;
    const uint64_t tb = frame ? sbk::k16_frame_tables_bytes(b->count, in_bytes) : sbk::k16_raw_tables_bytes(b->count, in_bytes);
    if (tables_bytes < tb || scratch_bytes < need) return 202;
    T t;
    memset(&t, 0, sizeof t);
    t.f.r.b = *b; t.f.idx = frame ? idx : nullptr;
    if (frame) sbk::k16_frame_carve(scratch, b->count, in_bytes, &t);
    else sbk::k16_raw_carve(scratch, b->count, in_bytes, &t);
    t.tables = (uint8_t*)tables; t.table_offs = table_offs; t.results = results;
    sbk::RawCompressPlan& q = t.f.r;
    memset(q.ctl, 0, sizeof(sbk::RawCompressCtl));
    auto blocks = [](uint64_t n, unsigned per) { return (unsigned)((n + per - 1) / per); };
    // K9 or K10, K1 with the CRC array
    sbemu::launch(blocks(b->count, 64), 64, 0, frame ? k10_plan_entry : k9_plan_entry, &t);
    sbemu::launch(blocks((uint64_t)b->count + 1, sbk::K4_TILE), sbk::K4_TILE, 128, scan_local_entry, &t);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry, &t);
    if (t.f.idx) {
        sbemu::launch(blocks((uint64_t)b->count + 1, sbk::K4_TILE), sbk::K4_TILE, 128, iscan_local_entry, &t);
        sbemu::launch(1, 1024, 1024 * 8, iscan_tiles_entry, &t);
    }
    sbemu::launch(blocks(q.nk, 64), 64, 0, frame ? k10_fill_entry : k9_fill_entry, &t);
    std::vector<uint64_t> rings((size_t)2 * 7 * sbk::K1_RING_GW, 0xCDCDCDCDCDCDCDCDull);
    uint32_t work = 0;
    K1Args k{sbk::k9_k1_batch(q), frame ? 1u : 0u, rings.data(), &work, t.f.crcs};
    sbemu::launch(2, 7 * 64, sbk::k1_multi_smem(7, 0), k1_entry, &k);
    sbemu::launch(blocks((uint64_t)q.nslot + 1, sbk::K4_TILE), sbk::K4_TILE, 128,
                  frame ? k10_bscan_local_entry : k9_bscan_local_entry, &t);
    sbemu::launch(1, 1024, 1024 * 8, bscan_tiles_entry, &t);
    sbemu::launch(2, 64, 0, frame ? k10_gather_entry : k9_gather_entry, &t);
    if (frame) sbemu::launch(2, 64, 0, k10_finish_entry, &t);
    else sbemu::launch(blocks(b->count, 64), 64, 0, k9_finish_entry, &t);
    // K16
    sbemu::launch(blocks((uint64_t)b->count + 1, sbk::K4_TILE), sbk::K4_TILE, 128,
                  frame ? frame_size_local_entry : raw_size_local_entry, &t);
    sbemu::launch(1, 1024, 1024 * 8, size_tiles_entry, &t);
    sbemu::launch(2, 64, 0, frame ? frame_export_entry : raw_export_entry, &t);
    return 0;
}

}

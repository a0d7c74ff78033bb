// emu_frame_index.cpp -- TEST TOOLING ONLY. The K7 chunk indexer (rust-snappy_b200/csrc/k7_frame_index.cuh) and the
// frame decoder's index-first path compiled by g++ against the fiber warp emulator, exposed to
// tests/test_frame_index_emu.py through a C interface. Built by that test into tests/emu/_build/libemu_frame_index.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k5_frame_decode.cuh"
#include "../../rust-snappy_b200/csrc/k7_frame_index.cuh"

static size_t up256(size_t v) { return (v + 255) / 256 * 256; }
static void k5_parse_entry(void* a) { sbk::k5_parse_body(*(sbk::DecodePlan*)a); }
static void k5_walk_entry(void* a) { sbk::k5_walk_body(*(sbk::DecodePlan*)a); }
static void k5_scan_local_entry(void* a) { sbk::k5_scan_local_body(*(sbk::DecodePlan*)a); }
static void k5_scan_tiles_entry(void* a) { sbk::k5_scan_tiles_body(*(sbk::DecodePlan*)a); }
static void k5_decode_entry(void* a) { sbk::k5_decode_body(*(sbk::DecodePlan*)a); }
static void k5_finish_entry(void* a) { sbk::k5_finish_body(*(sbk::DecodePlan*)a); }
static void k7_survivors_entry(void* a) { sbk::k7_survivors_body(*(sbk::IndexPlan*)a); }
static void k7_stitch_entry(void* a) { sbk::k7_stitch_body(*(sbk::IndexPlan*)a); }
static void k7_emit_entry(void* a) { sbk::k7_emit_body(*(sbk::IndexPlan*)a); }

// the launch sequence of launch_k7 in csrc/snapb200.cu
static void run_k7(sbk::IndexPlan p) {
    sbemu::launch(p.nseg ? (p.nseg + 3) / 4 : 1, 128, 0, k7_survivors_entry, &p);
    sbemu::launch(1, sbk::K7_STITCH_THREADS, sbk::K7_STITCH_SMEM, k7_stitch_entry, &p);
    sbemu::launch(p.nseg ? (p.nseg + 127) / 128 : 1, 128, 0, k7_emit_entry, &p);
}

extern "C" {

// sb_frame_index_device_ws under the emulator with segment length `seg` (0: default); *seg_out = the length used
int emu_frame_index(const uint8_t* in, uint64_t n, int fragment, uint64_t* index, uint32_t max_chunks, uint32_t* count,
                    uint64_t seg, uint64_t* seg_out) {
    const uint64_t segs = n / sbk::K7_SEG_MIN + 2;
    std::vector<sbk::K7Seg> table(segs);
    memset(table.data(), 0xCD, segs * sizeof(sbk::K7Seg));
    std::vector<uint32_t> meta(3 * segs, 0xCDCDCDCDu);
    const sbk::IndexPlan p = sbk::k7_make_plan(in, n, fragment ? 1u : 0u, max_chunks, seg ? seg : sbk::K7_SEG_DEFAULT,
                                               table.data(), segs, meta.data(), index, count);
    *seg_out = p.seg;
    run_k7(p);
    return 0;
}

// sb_frame_decode_device_ws without a caller index under the emulator, the kernel sequence of decode_index_phase and
// decode_payload_phase: K7 into the decode scratch -> parse over K7's count -> walk -> scan -> decode+CRC -> finish.
// *need_serial: whether the walk ran.
int emu_frame_decode_indexed(const uint8_t* in, uint64_t n, uint8_t* out, uint64_t cap, int fragment, sb_frame_result* result,
                             uint32_t max_chunks, uint64_t seg, uint32_t* need_serial) {
    std::vector<uint8_t> scratch(up256((size_t)max_chunks * sizeof(sbk::FChunk) + 64) + up256(((size_t)max_chunks + 1) * 8) +
                                 up256(((size_t)max_chunks / sbk::K4_TILE + 3) * 8) + up256((size_t)max_chunks * sizeof(sb_error) + 64) + 1024, 0xCD);
    uint8_t* q = (uint8_t*)up256((size_t)scratch.data());
    sbk::DecodePlan p;
    memset(&p, 0, sizeof p);
    p.in = in; p.n = n; p.fragment = fragment ? 1u : 0u;
    p.chunks = (sbk::FChunk*)q; q += up256((size_t)max_chunks * sizeof(sbk::FChunk) + 64);
    p.ooff = (uint64_t*)q; q += up256(((size_t)max_chunks + 1) * 8);
    p.tiles = (uint64_t*)q; q += up256(((size_t)max_chunks / sbk::K4_TILE + 3) * 8);
    p.statuses = (sb_error*)q; q += up256((size_t)max_chunks * sizeof(sb_error) + 64);
    p.ctl = (sbk::DecodeCtl*)q;
    p.cap_chunks = max_chunks; p.out = out; p.cap = cap; p.result = result;
    p.index = p.ooff; p.index_count = &p.ctl->index_count;
    memset(p.ctl, 0, sizeof(sbk::DecodeCtl));
    run_k7(sbk::k7_plan_for_decode(p, seg ? seg : sbk::K7_SEG_DEFAULT));
    sbemu::launch((max_chunks + 255) / 256, 256, 0, k5_parse_entry, &p);
    sbemu::launch(1, 32, 0, k5_walk_entry, &p);
    const unsigned ntiles = (max_chunks + sbk::K4_TILE - 1) / sbk::K4_TILE;
    sbemu::launch(ntiles ? ntiles : 1, sbk::K4_TILE, 128, k5_scan_local_entry, &p);
    sbemu::launch(1, 1024, 1024 * 8, k5_scan_tiles_entry, &p);
    sbemu::launch(3, 128, sbk::K3_TABLE_BYTES + 4 * sbk::K2_SMEM_PER_WARP, k5_decode_entry, &p);
    sbemu::launch(1, 32, 0, k5_finish_entry, &p);
    *need_serial = p.ctl->need_serial;
    return 0;
}

}

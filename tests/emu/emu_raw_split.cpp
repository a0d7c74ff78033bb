// emu_raw_split.cpp -- TEST TOOLING ONLY. K8's raw-stream split and block decode (rust-snappy_b200/csrc/k8_raw_split.cuh)
// compiled by g++ against the fiber warp emulator, exposed to tests/test_raw_split_emu.py through a C interface. Built
// by that test into tests/emu/_build/libemu_raw_split.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k8_raw_split.cuh"

static size_t up256(size_t v) { return (v + 255) / 256 * 256; }
static void header_entry(void* a) { sbk::k8_header_body(*(sbk::RawPlan*)a); }
static void chains_entry(void* a) { sbk::k8_chains_body(*(sbk::RawPlan*)a); }
static void merge_entry(void* a) { sbk::k8_merge_body(*(sbk::RawPlan*)a); }
static void stitch_entry(void* a) { sbk::k8_stitch_body(*(sbk::RawPlan*)a); }
static void counts_entry(void* a) { sbk::k8_counts_body(*(sbk::RawPlan*)a); }
static void scan_local_entry(void* a) { sbk::k8_scan_local_body(*(sbk::RawPlan*)a); }
static void scan_tiles_entry(void* a) { sbk::k8_scan_tiles_body(*(sbk::RawPlan*)a); }
static void cuts_entry(void* a) { sbk::k8_cuts_body(*(sbk::RawPlan*)a); }
static void blocks_entry(void* a) { sbk::k8_blocks_body(*(sbk::RawPlan*)a); }
static void fallback_entry(void* a) { sbk::k8_fallback_body(*(sbk::RawPlan*)a); }

extern "C" {

// sb_decompress_device_ws under the emulator: the scratch layout of make_raw_plan and the launch sequence of
// launch_raw_decode in csrc/snapb200.cu (with smaller grids). seg: segment length (0: default). Outputs: the cut table
// (65537 entries), *split_declined = the decline flag once the cuts are made (before any block is decoded), *seg_out.
int emu_raw_decode(const uint8_t* in, uint64_t n, uint8_t* out, uint64_t cap, sb_frame_result* result, uint64_t seg,
                   uint32_t* cuts, uint32_t* split_declined, uint64_t* seg_out) {
    const uint64_t segs = sbk::k8_max_segs(n);
    std::vector<uint8_t> scratch(256 + up256(((n >> 5) + 2) * 4) + 4 * up256(segs * 8) + up256(segs * 4) +
                                 up256((segs + 1) * 8) + up256((segs / sbk::K4_TILE + 3) * 8) +
                                 up256(((size_t)sbk::K8_MAX_BLOCKS + 1) * 4) + 512, 0xCD);
    uint8_t* q = (uint8_t*)up256((size_t)scratch.data());
    sbk::RawPlan p;
    memset(&p, 0, sizeof p);
    p.in = in; p.n = n; p.out = out; p.cap = cap; p.result = result;
    p.seg = sbk::k8_seg_len(seg);
    p.nseg = (uint32_t)((n + p.seg - 1) / p.seg);
    p.ctl = (sbk::RawCtl*)q; q += 256;
    p.marks = (uint32_t*)q; q += up256(((n >> 5) + 2) * 4);
    p.X = (uint64_t*)q; q += up256(segs * 8);
    p.Y = (uint64_t*)q; q += up256(segs * 8);
    p.ent = (uint64_t*)q; q += up256(segs * 8);
    p.ext = (uint64_t*)q; q += up256(segs * 8);
    p.cnt = (uint32_t*)q; q += up256(segs * 4);
    p.offs = (uint64_t*)q; q += up256((segs + 1) * 8);
    p.tiles = (uint64_t*)q; q += up256((segs / sbk::K4_TILE + 3) * 8);
    p.cut = (uint32_t*)q;
    memset(p.marks, 0, ((n >> 5) + 2) * 4);
    *seg_out = p.seg;
    const unsigned segw = p.nseg ? (p.nseg + 3) / 4 : 1;
    sbemu::launch(1, 32, 0, header_entry, &p);
    sbemu::launch(segw, 128, 0, chains_entry, &p);
    sbemu::launch(segw, 128, 0, merge_entry, &p);
    sbemu::launch(1, sbk::K8_STITCH_THREADS, sbk::K8_STITCH_THREADS * 16 + 16, stitch_entry, &p);
    sbemu::launch(segw, 128, 0, counts_entry, &p);
    const unsigned ntiles = (p.nseg + sbk::K4_TILE - 1) / sbk::K4_TILE;
    sbemu::launch(ntiles ? ntiles : 1, sbk::K4_TILE, 128, scan_local_entry, &p);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry, &p);
    sbemu::launch(segw, 128, 0, cuts_entry, &p);
    *split_declined = p.ctl->decline;
    memcpy(cuts, p.cut, ((size_t)sbk::K8_MAX_BLOCKS + 1) * 4);
    sbemu::launch(3, 128, 4 * sbk::K2_SMEM_PER_WARP, blocks_entry, &p);
    sbemu::launch(1, 32, sbk::K2_SMEM_PER_WARP, fallback_entry, &p);
    return 0;
}

}

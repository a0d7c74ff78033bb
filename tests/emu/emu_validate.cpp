// emu_validate.cpp -- TEST TOOLING ONLY. The validation bodies -- K2 with kStore = false, K8b's validate mode
// (rust-snappy_b200/csrc/k8_raw_split.cuh) and K19 (rust-snappy_b200/csrc/k19_validate.cuh) around K11's sequence --
// compiled by g++ against the fiber warp emulator, exposed to tests/test_validate_emu.py through a C interface. Built by
// that test into tests/emu/_build/libemu_validate.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k19_validate.cuh"

typedef sbk::RawBatchPlan RPlan;
typedef sbk::FrameDecodeBatchPlan FPlan;
typedef sbk::FrameValidatePlan VPlan;

// warp w of the grid checks units w, w + nwarps, ... with K2's output-free loop (no element table)
static void k2_entry(void* a) {
    const sb_batch& b = *(const sb_batch*)a;
    const unsigned wpb = sbk::block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)sbk::grid_dim() * wpb;
    for (uint64_t u = (uint64_t)sbk::block_idx() * wpb + sbk::warp_id(); u < b.count; u += nwarps) {
        const uint32_t i = (uint32_t)u;
        if (sbk::lane_id() == 0) b.out_lens[i] = 0;
        sbk::k2_decode_stream<true, false>(sbk::unit_in(b, i), sbk::unit_in_len(b, i), nullptr, sbk::unit_out_cap(b, i),
                                           &b.statuses[i], &b.out_lens[i], nullptr);
    }
}

static void plan_entry(void* a) { sbk::k8b_plan_body(*(RPlan*)a); }
static void plan_tiles_entry(void* a) { sbk::k8b_plan_tiles_body(*(RPlan*)a); }
static void chains_entry(void* a) { sbk::k8b_chains_body(*(RPlan*)a); }
static void merge_entry(void* a) { sbk::k8b_merge_body(*(RPlan*)a); }
static void stitch_entry(void* a) { sbk::k8b_stitch_body(*(RPlan*)a); }
static void counts_entry(void* a) { sbk::k8b_counts_body(*(RPlan*)a); }
static void scan_local_entry(void* a) { sbk::k8b_scan_local_body(*(RPlan*)a); }
static void scan_tiles_entry(void* a) { sbk::k8b_scan_tiles_body(*(RPlan*)a); }
static void cuts_entry(void* a) { sbk::k8b_cuts_body(*(RPlan*)a); }
static void vblocks_entry(void* a) { sbk::k8b_blocks_body<false>(*(RPlan*)a); }
static void vfinish_entry(void* a) { sbk::k8b_finish_body<false>(*(RPlan*)a); }

static void f_plan_entry(void* a) { sbk::k11_plan_body(*(FPlan*)a); }
static void f_plan_tiles_entry(void* a) { sbk::k11_plan_tiles_body(*(FPlan*)a); }
static void f_survivors_entry(void* a) { sbk::k11_survivors_body(*(FPlan*)a); }
static void f_stitch_entry(void* a) { sbk::k11_stitch_body(*(FPlan*)a); }
static void f_link_entry(void* a) { sbk::k11_link_body(*(FPlan*)a); }
static void f_count_entry(void* a) { sbk::k11_count_body(*(FPlan*)a); }
static void f_range_tiles_entry(void* a) { sbk::k11_range_tiles_body(*(FPlan*)a); }
static void f_emit_entry(void* a) { sbk::k11_emit_body(*(FPlan*)a); }
static void f_parse_entry(void* a) { sbk::k11_parse_body(*(FPlan*)a); }
static void f_fill_entry(void* a) { sbk::k11_fill_body(*(FPlan*)a); }
static void f_oscan_local_entry(void* a) { sbk::k11_oscan_local_body(*(FPlan*)a); }
static void f_oscan_tiles_entry(void* a) { sbk::k11_oscan_tiles_body(*(FPlan*)a); }
static void f_validate_entry(void* a) { sbk::k19_validate_body(*(VPlan*)a); }
static void f_finish_entry(void* a) { sbk::k11_finish_body(*(FPlan*)a); }

// validate_view of csrc/snapb200.cu: inputs and results only, caps of 2^32 - 1
static sb_batch view(const sb_batch& b) {
    sb_batch u;
    memset(&u, 0, sizeof u);
    u.in_ptrs = b.in_ptrs; u.in_base = b.in_base; u.in_stride = b.in_stride; u.in_lens = b.in_lens;
    u.in_len_uniform = b.in_len_uniform; u.out_cap_uniform = 0xFFFFFFFFu;
    u.out_lens = b.out_lens; u.statuses = b.statuses; u.count = b.count;
    return u;
}

extern "C" {

// K2 with kStore = false over every unit (out_caps as given), one warp per unit, `grid` CTAs of 64 threads
void emu_k2_validate(const sb_batch* b, unsigned grid) { sbemu::launch(grid, 64, 0, k2_entry, (void*)b); }

uint64_t emu_raw_validate_scratch_bytes(uint32_t count, uint64_t in_bytes) { return sbk::k8b_carve(nullptr, count, in_bytes, nullptr); }

// sb_validate_batch_device_ws under the emulator: the call checks, the view, the scratch layout of k8b_carve and the
// launch sequence of launch_raw_validate in csrc/snapb200.cu, with small grids. seg: segment length (0: the default).
int emu_raw_validate_batch(const sb_batch* b, uint64_t in_bytes, uint32_t* unit_blocks, void* scratch, uint64_t scratch_bytes,
                           uint64_t seg) {
    if (!b || !b->out_lens || !b->statuses || !scratch || b->count >= sbk::K8B_MAX_COUNT) return 202;
    if (b->count == 0) return 0;
    if (scratch_bytes < sbk::k8b_carve(nullptr, b->count, in_bytes, nullptr)) return 202;
    RPlan q;
    memset(&q, 0, sizeof q);
    q.b = view(*b); q.seg = sbk::k8_seg_len(seg); q.unit_blocks = unit_blocks;
    sbk::k8b_carve(scratch, b->count, in_bytes, &q);
    memset(q.bctl, 0, sizeof(sbk::RawBatchCtl));
    const unsigned utiles = (unsigned)(((uint64_t)b->count + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(utiles, sbk::K4_TILE, 128, plan_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, plan_tiles_entry, &q);
    sbemu::launch(3, 128, 0, chains_entry, &q);
    sbemu::launch(3, 128, 0, merge_entry, &q);
    sbemu::launch(b->count < 3 ? b->count : 3, sbk::K8_STITCH_THREADS, sbk::K8_STITCH_THREADS * 16 + 16, stitch_entry, &q);
    sbemu::launch(3, 128, 0, counts_entry, &q);
    const unsigned ctiles = (unsigned)(((uint64_t)q.nseg_cap + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(ctiles, sbk::K4_TILE, 128, scan_local_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry, &q);
    sbemu::launch(3, 128, 0, cuts_entry, &q);
    sbemu::launch(3, 128, 4 * sbk::K2_SMEM_PER_WARP, vblocks_entry, &q);
    sbemu::launch(2, 128, 4 * sbk::K2_SMEM_PER_WARP, vfinish_entry, &q);
    return 0;
}

uint64_t emu_frame_validate_scratch_bytes(uint32_t count, uint64_t in_bytes, uint32_t max_chunks) {
    return sbk::k19_carve(nullptr, count, in_bytes, max_chunks, nullptr);
}

// sb_frame_validate_batch_device_ws under the emulator: the call checks, the view, the scratch layout of k19_carve and
// the launch sequence of launch_frame_validate_batch in csrc/snapb200.cu, with small grids (K19's grid holds fewer warps
// than slots, so warps take several chunks). seg: K7 segment length (0: the library's default).
int emu_frame_validate_batch(const sb_batch* b, uint64_t in_bytes, uint32_t flags, const uint64_t* cidx, const uint64_t* cidx_at,
                             uint32_t max_chunks, uint32_t* unit_chunks, void* scratch, uint64_t scratch_bytes, uint64_t seg) {
    if (!b || !b->out_lens || !b->statuses || !scratch || b->count >= sbk::K11_MAX_COUNT || !cidx != !cidx_at) return 202;
    if (max_chunks == 0 || max_chunks > sbk::K11_MAX_CHUNKS) return 202;
    if (b->count == 0) return 0;
    if (scratch_bytes < sbk::k19_carve(nullptr, b->count, in_bytes, max_chunks, nullptr)) return 202;
    VPlan t;
    memset(&t, 0, sizeof t);
    FPlan& q = t.q;
    q.b = view(*b); q.fragment = flags & 1u; q.cidx = cidx; q.cidx_at = cidx_at; q.unit_chunks = unit_chunks;
    q.seg = seg ? (seg < sbk::K7_SEG_MIN ? sbk::K7_SEG_MIN : seg) : sbk::K7_SEG_DEFAULT;
    sbk::k19_carve(scratch, b->count, in_bytes, max_chunks, &t);
    const unsigned utiles = (unsigned)(((uint64_t)b->count + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const unsigned stiles = (unsigned)(((uint64_t)max_chunks + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    *q.in_total = 0;
    sbemu::launch(utiles, sbk::K4_TILE, 128, f_plan_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, f_plan_tiles_entry, &q);
    if (cidx) {
        sbemu::launch(2, 64, 0, f_link_entry, &q);
    } else {
        sbemu::launch(2, 64, 0, f_survivors_entry, &q);
        sbemu::launch(b->count < 3 ? b->count : 3, sbk::K7_STITCH_THREADS, sbk::K7_STITCH_SMEM, f_stitch_entry, &q);
    }
    sbemu::launch(utiles, sbk::K4_TILE, 128, f_count_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, f_range_tiles_entry, &q);
    if (!cidx) sbemu::launch(2, 32, 0, f_emit_entry, &q);
    sbemu::launch(2, 64, 0, f_parse_entry, &q);
    sbemu::launch(2, 32, 0, f_fill_entry, &q);
    sbemu::launch(stiles, sbk::K4_TILE, 128, f_oscan_local_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, f_oscan_tiles_entry, &q);
    const unsigned vgrid = t.nslots < 8 ? 1 : 2;                       // at most 8 warps: each takes several chunks
    *t.next = 0;
    sbemu::launch(vgrid, 128, sbk::K3_TABLE_BYTES + 4 * sbk::K2_SMEM_PER_WARP, f_validate_entry, &t);
    sbemu::launch(2, 32, 0, f_finish_entry, &q);
    return 0;
}

}

// emu_crc_copy.cpp -- TEST TOOLING ONLY. K3's two warp CRC-32C variants (rust-snappy_b200/csrc/k3_crc32c.cuh), the warp
// copy of common.cuh and the two-level scan of k4_frame.cuh compiled by g++ against the fiber warp emulator, exposed to
// tests/test_crc_copy_emu.py through a C interface. Built by that test into tests/emu/_build/libemu_crc_copy.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k3_crc32c.cuh"
#include "../../rust-snappy_b200/csrc/k4_frame.cuh"

#include <sys/mman.h>
#include <unistd.h>

namespace {

static void k3_crc_entry(void* a) { sbk::k3_crc_body(*(sb_batch*)a); }

struct Crc1Args { const uint64_t* ptrs; const uint32_t* lens; uint32_t count; uint32_t* out; };
// K1's emitter form: the CTA builds the byte table, then warp w checksums units w, w + nwarps, ...
static void k3_crc1_entry(void* a) {
    const Crc1Args* x = (const Crc1Args*)a;
    uint32_t* tab = (uint32_t*)sbk::smem();
    sbk::k3_build_table1(tab, sbk::thread_idx(), sbk::block_dim());
    sbk::syncthreads();
    const unsigned nw = sbk::block_dim() >> 5;
    for (uint32_t i = sbk::warp_id(); i < x->count; i += nw) {
        const uint32_t crc = sbk::k3_warp_crc32c_masked1(tab, (const uint8_t*)x->ptrs[i], x->lens[i]);
        if (sbk::lane_id() == 0) x->out[i] = crc;
    }
}

struct CopyArgs { const uint64_t* jobs; uint32_t count; int ef; };
// one warp runs the (dst, src, n) jobs in order
static void copy_entry(void* a) {
    const CopyArgs* x = (const CopyArgs*)a;
    for (uint32_t i = 0; i < x->count; i++) {
        uint8_t* dst = (uint8_t*)x->jobs[3 * i];
        const uint8_t* src = (const uint8_t*)x->jobs[3 * i + 1];
        const uint32_t n = (uint32_t)x->jobs[3 * i + 2];
        if (x->ef) sbk::warp_copy_t<true>(dst, src, n);
        else sbk::warp_copy_t<false>(dst, src, n);
    }
}

struct ScanArgs { uint32_t count; const uint32_t* vals; uint64_t* offs; uint64_t* tiles; uint64_t base; };
static void scan_local_entry(void* a) {
    const ScanArgs* x = (const ScanArgs*)a;
    sbk::scan_local_body(x->count, [&](uint32_t i) { return x->vals[i]; }, x->offs, x->tiles);
}
static void scan_tiles_entry(void* a) {
    const ScanArgs* x = (const ScanArgs*)a;
    sbk::scan_tiles_body(x->count, x->base, x->tiles);
}

}  // namespace

extern "C" {

// sb_crc32c_masked_batch_device under the emulator: k3_crc_body over the batch, `grid` CTAs of 4 warps
int emu_crc_batch(const sb_batch* b, unsigned grid) {
    sb_batch c = *b;
    sbemu::launch(grid, 128, sbk::K3_TABLE_BYTES, k3_crc_entry, &c);
    return 0;
}

// k3_warp_crc32c_masked1 (the single-table variant K1 fuses into frame encode) over units ptrs[i] / lens[i]
int emu_crc1(const uint64_t* ptrs, const uint32_t* lens, uint32_t count, uint32_t* out) {
    Crc1Args a{ptrs, lens, count, out};
    sbemu::launch(1, 64, sbk::K3_TABLE1_BYTES, k3_crc1_entry, &a);
    return 0;
}

// warp_copy_t<ef> of every (dst, src, n) triple in jobs[3 * count], one after another
int emu_warp_copy(const uint64_t* jobs, uint32_t count, int ef) {
    CopyArgs a{jobs, count, ef};
    sbemu::launch(1, 32, 0, copy_entry, &a);
    return 0;
}

// warp_copy_t<ef>(dst, src, n) with `data` placed between inaccessible pages: at_start = 0 puts the source's last byte
// right before a PROT_NONE page, at_start = 1 puts its first byte right after one. A load outside [src, src + n) that
// crosses the page boundary faults. Returns the source address's offset mod 16, or -1 if the mapping failed.
int emu_warp_copy_fenced(const uint8_t* data, uint32_t n, uint8_t* dst, int ef, int at_start) {
    const size_t pg = (size_t)sysconf(_SC_PAGESIZE);
    const size_t body = (n + pg - 1) / pg * pg + pg;
    uint8_t* m = (uint8_t*)mmap(nullptr, body + 2 * pg, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (m == MAP_FAILED) return -1;
    uint8_t* fence = at_start ? m : m + pg + body;
    uint8_t* src = at_start ? m + pg : fence - n;
    memcpy(src, data, n);
    int rc = mprotect(fence, pg, PROT_NONE);
    if (rc == 0) {
        const uint64_t job[3] = {(uint64_t)(uintptr_t)dst, (uint64_t)(uintptr_t)src, n};
        emu_warp_copy(job, 1, ef);
    }
    const int mod = (int)((uintptr_t)src & 15u);
    munmap(m, body + 2 * pg);
    return rc == 0 ? mod : -1;
}

// the two-level scan of K4/K5 over vals[0..count): tile-local scans of K4_TILE threads, then scan_tiles_body with
// `tiles_threads` threads (the kernels use 1024; fewer makes one thread sum several tiles at a small count)
int emu_scan(uint32_t count, const uint32_t* vals, uint64_t base, uint64_t* offs, uint64_t* tiles, unsigned tiles_threads) {
    ScanArgs a{count, vals, offs, tiles, base};
    const unsigned ntiles = (count + sbk::K4_TILE - 1) / sbk::K4_TILE;
    sbemu::launch(ntiles ? ntiles : 1, sbk::K4_TILE, 32 * sizeof(uint32_t), scan_local_entry, &a);
    sbemu::launch(1, tiles_threads, tiles_threads * sizeof(uint64_t), scan_tiles_entry, &a);
    return 0;
}

}

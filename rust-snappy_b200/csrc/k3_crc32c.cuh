// k3_crc32c.cuh -- K3: masked CRC-32C per chunk, one chunk per warp.
//
// Replaces reference src/crc32.rs:35-38 (crc32c_masked) and :59-111 (the SSE4.2
// and slicing-by-16 bodies), tables of build.rs:69-124 (poly 0x82F63B78).
//
// A CRC is linear over GF(2): the warp cuts the chunk into 32 slices, every
// lane runs a slicing-by-4 table CRC over its slice (tables in shared memory),
// each partial state is advanced over "the bytes that follow it" by one
// polynomial multiplication with x^(8*bytes) mod P, and the partials are XORed.
#pragma once
#include "common.cuh"

namespace sbk {

static const uint32_t K3_POLY = 0x82F63B78u;
static const uint32_t K3_TABLE_BYTES = 4 * 256 * 4;

// a(x)*b(x) mod P, reflected bit order (bit 31 = x^0)
SB_DEVICE uint32_t k3_mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
#pragma unroll 4
    for (int i = 0; i < 32; i++) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b & 1u) ? (b >> 1) ^ K3_POLY : b >> 1;
    }
    return p;
}

// x^(8*nbytes) mod P
SB_DEVICE uint32_t k3_xpow8(uint32_t nbytes) {
    uint32_t r = 0x80000000u;      // x^0
    uint32_t sq = 0x00800000u;     // x^8
    while (nbytes) {
        if (nbytes & 1u) r = k3_mulmod(sq, r);
        sq = k3_mulmod(sq, sq);
        nbytes >>= 1;
    }
    return r;
}

// Build the 4 slicing tables in shared memory (all threads of the CTA).
SB_DEVICE void k3_build_tables(uint32_t* tab) {
    for (uint32_t i = thread_idx(); i < 256; i += block_dim()) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ K3_POLY : c >> 1;
        tab[i] = c;
    }
    syncthreads();
    for (uint32_t i = thread_idx(); i < 256; i += block_dim()) {
        uint32_t c = tab[i];
        for (int j = 1; j < 4; j++) { c = (c >> 8) ^ tab[c & 0xFFu]; tab[j * 256 + i] = c; }
    }
    syncthreads();
}

SB_DEVICE uint32_t k3_bytes(const uint32_t* tab, uint32_t st, const uint8_t* p, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) st = tab[(st ^ p[i]) & 0xFFu] ^ (st >> 8);
    return st;
}

// raw CRC state over [p, p+n) starting from st
SB_DEVICE uint32_t k3_slice(const uint32_t* tab, uint32_t st, const uint8_t* p, uint32_t n) {
    uint32_t head = (uint32_t)((0 - (uintptr_t)p) & 3u);
    if (head > n) head = n;
    st = k3_bytes(tab, st, p, head);
    p += head; n -= head;
    const uint32_t* w = (const uint32_t*)p;
    const uint32_t nw = n >> 2;
    for (uint32_t i = 0; i < nw; i++) {
        const uint32_t v = st ^ w[i];
        st = tab[768 + (v & 0xFFu)] ^ tab[512 + ((v >> 8) & 0xFFu)] ^ tab[256 + ((v >> 16) & 0xFFu)] ^ tab[v >> 24];
    }
    return k3_bytes(tab, st, p + 4 * nw, n & 3u);
}

// masked CRC-32C of [p, p+n) computed by the calling warp; result in all lanes
SB_DEVICE uint32_t k3_warp_crc32c_masked(const uint32_t* tab, const uint8_t* p, uint32_t n) {
    const unsigned lane = lane_id();
    // slice length ceil(n/32) rounded up to a multiple of 4; as ((n - 1) >> 5) + 1 it cannot wrap near 2^32 like n + 31
    // (n = 0 gives a huge slice, but every slice is clipped to [0, n) and stays empty)
    uint32_t sl = (((n - 1) >> 5) + 4) & ~3u;
    if (sl < 64) sl = 64;
    uint64_t b0 = (uint64_t)lane * sl, b1 = b0 + sl;
    if (b0 > n) b0 = n;
    if (b1 > n) b1 = n;
    uint32_t st = (lane == 0) ? 0xFFFFFFFFu : 0u;
    st = k3_slice(tab, st, p + b0, (uint32_t)(b1 - b0));
    const uint32_t after = n - (uint32_t)b1;
    if (after && st) st = k3_mulmod(k3_xpow8(after), st);
#pragma unroll
    for (int k = 16; k >= 1; k >>= 1) st ^= shfl_xor(st, k);
    const uint32_t crc = ~st;
    return ((crc >> 15) | (crc << 17)) + 0xA282EAD8u;   // src/crc32.rs:35-38
}

// ---- single-table variant for kernels that can spare only 1 KB of shared memory (K1's emitter warps:
// frame encode computes the chunk checksum beside the compress call, reference src/frame.rs:76)
static const uint32_t K3_TABLE1_BYTES = 256 * 4;
// threads [t0, t0+nt) of the CTA build the byte table; the caller synchronises afterwards
SB_DEVICE void k3_build_table1(uint32_t* tab, unsigned t, unsigned nt) {
    for (uint32_t i = t; i < 256; i += nt) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (c >> 1) ^ K3_POLY : c >> 1;
        tab[i] = c;
    }
}
SB_DEVICE uint32_t k3_word1(const uint32_t* tab, uint32_t st, uint32_t w) {
    st ^= w;
    st = tab[st & 0xFFu] ^ (st >> 8);
    st = tab[st & 0xFFu] ^ (st >> 8);
    st = tab[st & 0xFFu] ^ (st >> 8);
    return tab[st & 0xFFu] ^ (st >> 8);
}
// raw CRC state over [p, p+n) with the byte table: 16-byte loads once p is 16-byte aligned
SB_DEVICE uint32_t k3_slice1(const uint32_t* tab, uint32_t st, const uint8_t* p, uint32_t n) {
    uint32_t head = (uint32_t)((0 - (uintptr_t)p) & 15u);
    if (head > n) head = n;
    st = k3_bytes(tab, st, p, head);
    p += head; n -= head;
    const uint4* v = (const uint4*)p;
    const uint32_t nv = n >> 4;
    for (uint32_t i = 0; i < nv; i++) {
        const uint4 q = v[i];
        st = k3_word1(tab, st, q.x); st = k3_word1(tab, st, q.y); st = k3_word1(tab, st, q.z); st = k3_word1(tab, st, q.w);
    }
    return k3_bytes(tab, st, p + 16 * nv, n & 15u);
}
// masked CRC-32C of [p, p+n) by the calling warp with the byte table; result in all lanes
SB_DEVICE uint32_t k3_warp_crc32c_masked1(const uint32_t* tab, const uint8_t* p, uint32_t n) {
    const unsigned lane = lane_id();
    uint32_t sl = (((n - 1) >> 5) + 16) & ~15u;    // ceil(n/32) rounded up to a multiple of 16, without wrapping (see k3_warp_crc32c_masked)
    if (sl < 64) sl = 64;
    uint64_t b0 = (uint64_t)lane * sl, b1 = b0 + sl;
    if (b0 > n) b0 = n;
    if (b1 > n) b1 = n;
    uint32_t st = (lane == 0) ? 0xFFFFFFFFu : 0u;
    st = k3_slice1(tab, st, p + b0, (uint32_t)(b1 - b0));
    const uint32_t after = n - (uint32_t)b1;
    if (after && st) st = k3_mulmod(k3_xpow8(after), st);
#pragma unroll
    for (int k = 16; k >= 1; k >>= 1) st ^= shfl_xor(st, k);
    const uint32_t crc = ~st;
    return ((crc >> 15) | (crc << 17)) + 0xA282EAD8u;   // src/crc32.rs:35-38
}

// Kernel body: warp w handles units w, w+nwarps, ...; out_lens[i] receives the masked CRC.
SB_DEVICE void k3_crc_body(const BatchDesc& b) {
    uint32_t* tab = (uint32_t*)smem();
    k3_build_tables(tab);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t u = (uint64_t)block_idx() * wpb + warp_id(); u < b.count; u += nwarps) {
        const uint32_t i = (uint32_t)u;
        const uint32_t crc = k3_warp_crc32c_masked(tab, unit_in(b, i), unit_in_len(b, i));
        if (lane_id() == 0) b.out_lens[i] = crc;
    }
}

}  // namespace sbk

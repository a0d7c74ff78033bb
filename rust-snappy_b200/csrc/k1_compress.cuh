// k1_compress.cuh -- K1: batched raw Snappy block encode, bit-exact with the reference encoder.
//
// Replaces reference src/compress.rs:195-317 (Block::compress), :323-369
// (emit_copy/emit_copy2), :378-412 (extend_match), :417-426 (done), :433-474
// (emit_literal), :491-526 (block_table + hash) and, per unit, the varint
// header + block loop of Encoder::compress (:119-153).
//
// The greedy parse is a serial dependency chain (every table insert depends on
// every earlier match decision), so bit-exactness forbids a "better" parallel
// match finder. One CTA per SM hosts several independent chains; a chain is a
// pair of warps working on one <=64KB block that is read in place from global
// memory / L2, with its 16K-entry u16 hash table in shared memory (7 chains) or in
// an L2-resident global scratch (the others):
//
//  * PARSER warp. Looks at 64 consecutive positions per step, two per lane. Every
//    lane hashes its positions, reads the table as of the step start, fetches the
//    candidates and computes "would a probe here hit, and how long is the match".
//    From the hit bitmask each hit position computes where the NEXT copy would start
//    (rematch hit at the copy end, else the first later hit of the scan), pointer
//    doubling from the step's entry state yields the copies the serial encoder
//    takes, and the inserted positions are "everything except copy interiors".
//    The inserts are committed; if two inserted positions collided on a slot, the
//    step is accepted up to the first position whose candidate should have come from
//    inside the step and restarts there.
//  * serial path: the reference's control flow executed by the warp (scan probes
//    32 at a time with match.any conflict resolution, 128-byte match extension).
//    Used for scan runs past 32 probes (stride > 1) and the block tail.
//  * EMITTER warp. Consumes the parser's (position, length, offset) copy events
//    from a ring, 32 at a time: literal/copy tag sizes, a warp scan for output
//    offsets, tags and literal bytes written straight to HBM (evict-first).
//
// Tried and rejected (slower on hardware): 32-position steps, unaligned windows,
// speculative slot reads for the L2-table chains, an mbarrier wake-up for the emitter, and a second-generation parser
// with exact windows and pipelined candidate evaluation. The one-pair-per-CTA layouts of round 1 (shared-memory window, pipelined parser
// warps) are gone as well (DESIGN.md section 4).
#pragma once
#include "common.cuh"
#include "k3_crc32c.cuh"

#if defined(K1_PROFILE) && defined(__CUDACC__)
// Optional phase timers for kernel archaeology (tools/k1_phase_profile.sh builds a separate
// library with -DK1_PROFILE; the product build has none of this).
// [0..11]: cycles per phase (K1_TICK slots), [12 + s]: parser warps per scheduler, [16 + k]: K1_COUNT(k) steps
__device__ unsigned long long g_k1_prof[18];
#define K1_TICK(slot) do { const long long _now = clock64(); if (sbk::lane_id() == 0) k1_acc[slot] += (unsigned long long)(_now - k1_t0); k1_t0 = _now; } while (0)
#define K1_COUNT(k) do { if (sbk::lane_id() == 0) k1_acc[12 + (k)]++; } while (0)
#define K1_PROF_DECL unsigned long long k1_acc[14] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0}; long long k1_t0 = clock64();
#define K1_PROF_ARGS , unsigned long long* k1_acc, long long& k1_t0
#define K1_PROF_PASS , k1_acc, k1_t0
#define K1_PROF_FLUSH do { if (sbk::lane_id() == 0) for (int _i = 0; _i < 14; _i++) atomicAdd(&g_k1_prof[_i < 12 ? _i : _i + 4], k1_acc[_i]); } while (0)
// [12 + s]: parser warps the hardware placed on scheduler s (%warpid & 3), one count per warp and launch
#define K1_PROF_CENSUS(is_parser) do { unsigned _hw; asm volatile("mov.u32 %0, %%warpid;" : "=r"(_hw)); \
    if ((is_parser) && sbk::lane_id() == 0) atomicAdd(&g_k1_prof[12 + (_hw & 3u)], 1ull); } while (0)
#else
#define K1_PROF_CENSUS(is_parser) do { } while (0)
#define K1_TICK(slot) do { } while (0)
#define K1_PROF_DECL
#define K1_PROF_ARGS
#define K1_PROF_PASS
#define K1_PROF_FLUSH do { } while (0)
#if defined(SB_EMU)
// CPU warp-emulator build (tests/emu): the same step counts, readable by the tests through the symbol
extern "C" { __attribute__((weak)) unsigned long long sb_emu_k1_windows[4]; }
#define K1_COUNT(k) do { if (sbk::lane_id() == 0) sb_emu_k1_windows[k]++; } while (0)
#else
#define K1_COUNT(k) do { } while (0)
#endif
#endif
// K1_COUNT: [0] fast-path steps whose probe the previous step issued (hoisted), [1] probes issued at the loop top;
// emulator build only: [2] probes with a table slot that changed between the read and the use, [3] sequential-word
// fetches that reach byte n of the block (both must stay 0)

namespace sbk {

static const uint32_t K1_TABLE_BYTES = 32768;                // 16K-entry u16 table
static const uint32_t K1_RING_GW = 256;                      // copy events in flight per chain (global scratch, L2 resident)

// 4 bytes at win+p through two aligned word loads. `win` may be a shared-memory window
// (4-byte aligned) or the unit's input in global memory (any alignment): the loads are
// aligned on the absolute address.
SB_DEVICE uint32_t k1_rd32(const uint8_t* win, uint32_t p) {
    const uintptr_t a = (uintptr_t)(win + p);
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    return funnel_r(w[0], w[1], (unsigned)(a & 3u) * 8);
}
// same, but never touches a byte at or beyond win+n (zero fill): for positions near the end
SB_DEVICE uint32_t k1_rd32_end(const uint8_t* win, uint32_t p, uint32_t n) {
    if (p + 8 <= n) return k1_rd32(win, p);
    uint32_t v = 0;
    for (uint32_t k = 0; k < 4; k++) if (p + k < n) v |= (uint32_t)win[p + k] << (8 * k);
    return v;
}

// ---------------------------------------------------------------- event ring
struct K1Ring {
    uint64_t* ev;        // `size` entries (power of two)
    uint32_t* ctrl;      // [0]=head (produced), [1]=tail (consumed), [6..7]=producer counters between units, [8]=unit
    uint32_t size;
};
// pos | len << 17 | off << 34, built as its two 32-bit halves (pos, len <= 65536: len << 17 carries into the high word)
SB_DEVICE uint64_t k1_event(uint32_t pos, uint32_t len, uint32_t off) {
    return (uint64_t)(pos | (len << 17)) | ((uint64_t)((len >> 15) | (off << 2)) << 32);
}
// producer side. The parser keeps private copies of the ring counters and only
// touches the shared ones when it has to: `tail_seen` is refreshed when the ring
// looks full, `head` is published every K1_PUBLISH events (the emitter works on
// fuller batches and the parser pays one fence per batch instead of one per step).
struct K1Prod {
    uint32_t head;        // events written so far
    uint32_t published;   // value of ctrl[0]
    uint32_t tail_seen;   // last value read from ctrl[1]
};
static const uint32_t K1_PUBLISH = 64;   // a publish costs a CTA fence behind global stores (~0.5k cycles): amortise it

SB_DEVICE void k1_publish(const K1Ring& r, K1Prod& pr) {
    if (pr.published == pr.head) return;
    threadfence_block();                                  // EVERY lane fences its own event stores (CTA scope) ...
    syncwarp();                                           // ... before lane 0 makes the new head visible
    if (lane_id() == 0) st_volatile(&r.ctrl[0], pr.head);
    pr.published = pr.head;
}
SB_DEVICE void k1_wait_space(const K1Ring& r, K1Prod& pr, uint32_t need) {
    if (pr.head + need - pr.tail_seen <= r.size) return;
    k1_publish(r, pr);                                   // the emitter must see everything before we wait on it
    for (;;) {
        pr.tail_seen = shfl(ld_volatile(&r.ctrl[1]), 0);   // one reader: the decision must be warp-uniform
        if (pr.head + need - pr.tail_seen <= r.size) return;
        spin();
    }
}
SB_DEVICE void k1_push(const K1Ring& r, K1Prod& pr, uint64_t e) {
    k1_wait_space(r, pr, 1);
    if (lane_id() == 0) r.ev[pr.head & (r.size - 1)] = e;
    pr.head++;
    if (pr.head - pr.published >= K1_PUBLISH) k1_publish(r, pr);
}

// ------------------------------------------------------------- serial pieces
// match extension from (s, c) to the END OF THE BLOCK (src/compress.rs:378-412)
SB_DEVICE uint32_t k1_extend(const uint8_t* win, uint32_t n, uint32_t s, uint32_t c) {
    const unsigned lane = lane_id();
    for (;;) {
        const uint32_t p = s + 4 * lane;
        uint32_t m = 0;
        if (p < n) {
            const uint32_t avail = n - p;
            // the candidate side sits below p, but its aligned two-word read may reach 6 bytes past it: near the end of
            // the block (= possibly the end of the caller's allocation) both sides use the bounded read
            const uint32_t x = k1_rd32_end(win, p, n) ^ (p + 8 <= n ? k1_rd32(win, c + 4 * lane) : k1_rd32_end(win, c + 4 * lane, n));
            m = x ? (uint32_t)(ffs(x) - 1) >> 3 : 4;
            if (m > avail) m = avail;
        }
        const uint32_t stop = ballot(m < 4);
        if (!stop) { s += 128; c += 128; continue; }
        const unsigned f = ffs(stop) - 1;
        return s + 4 * f + shfl(m, f);
    }
}

struct K1State {
    uint32_t s;        // next event position
    uint32_t skip;     // scan state (src/compress.rs:204-211); meaningful when !rematch
    bool rematch;      // true: a copy just ended at s and s-1 is already inserted (:285-301 first half)
};
// the step at w (holding st.s) runs on the parser's fast path: well inside the block (every position up to w + 63
// may be probed, and the words it reads end before byte n), and a scan still probes every position
SB_DEVICE bool k1_fast(uint32_t w, const K1State& st, uint32_t s_limit) {
    return w + 68 < s_limit && (st.rematch || st.skip < 64);
}

#define K1_HASH(x) (((uint32_t)(x) * 0x1E35A7BDu) >> shift)
// after a copy ends at e: `if s >= s_limit return` else insert e-1 (:275-295)
SB_DEVICE void k1_preinsert(const uint8_t* win, uint16_t* table, unsigned shift, uint32_t s_limit, uint32_t e) {
    if (e < s_limit) {
        const uint32_t h = K1_HASH(k1_rd32(win, e - 1));
        syncwarp();
        if (lane_id() == 0) table[h] = (uint16_t)(e - 1);
        syncwarp();
    }
}

// The reference's control flow, one event (or one 32-probe scan batch) at a time,
// until the parse position reaches `target` or the block is finished.
// Returns true when the block is finished.
SB_DEVICE bool k1_serial(const uint8_t* win, uint32_t n, uint16_t* table, unsigned shift, uint32_t s_limit,
                         K1State& st, uint32_t target, const K1Ring& ring, K1Prod& head) {
    const unsigned lane = lane_id();
    for (;;) {
        uint32_t cand;
        if (st.rematch) {
            if (st.s >= s_limit) return true;
            // probe at s (:296-313); s-1 was inserted when the copy ended
            const uint32_t cur = k1_rd32(win, st.s);
            const uint32_t h = K1_HASH(cur);
            cand = table[h];
            syncwarp();
            if (lane == 0) table[h] = (uint16_t)st.s;
            syncwarp();
            if (cur != k1_rd32(win, cand)) {
                st.s += 1; st.rematch = false; st.skip = 32;
                if (st.s >= target) return false;
                continue;
            }
        } else {
            // scan: 32 probes per step (:204-245)
            uint32_t pos = st.s, sk = st.skip;
            if (st.skip == 32) { pos = st.s + lane; sk = 32 + lane; }
            else { for (unsigned i = 0; i < lane; i++) { const uint32_t step = sk >> 5; pos += step; sk += step; } }
            const uint32_t step = sk >> 5;
            const bool valid = pos + step <= s_limit;          // probe happens only if s_next <= s_limit
            uint32_t cur = 0, h = 0xFFFFFFFFu - lane, c = 0;   // invalid lanes get unique pseudo-hashes
            if (valid) { cur = k1_rd32(win, pos); h = K1_HASH(cur); c = table[h]; }
            const uint32_t same = match_any(h);
            const uint32_t below = same & ((1u << lane) - 1u);
            const uint32_t prev_pos = shfl(pos, below ? 31 - clz(below) : 0);
            if (below) c = prev_pos;                            // an earlier probe of this batch inserted first
            const bool hit = valid && cur == k1_rd32(win, c);
            const uint32_t hm = ballot(hit), vm = ballot(valid);
            const unsigned fi = vm == 0xFFFFFFFFu ? 32 : ffs(~vm) - 1;
            const unsigned fh = hm ? ffs(hm) - 1 : 32;
            const unsigned ncommit = fh < fi ? fh + 1 : fi;    // lanes [0, ncommit) perform their insert
            syncwarp();                                         // probe reads precede the batch's inserts
            if (lane < ncommit) {
                const uint32_t later = same & ~((2u << lane) - 1u) & (ncommit >= 32 ? 0xFFFFFFFFu : ((1u << ncommit) - 1u));
                if (!later) table[h] = (uint16_t)pos;           // last writer of a slot wins
            }
            syncwarp();
            if (fh >= fi) {
                if (fi < 32) return true;                       // ran past s_limit: block is finished
                st.s = shfl(pos + step, 31);
                st.skip = shfl(sk + step, 31);
                if (st.s >= target) return false;
                continue;
            }
            st.s = shfl(pos, fh);
            cand = shfl(c, fh);
        }
        // copy (:258-276)
        const uint32_t base = st.s;
        const uint32_t end = k1_extend(win, n, base + 4, cand + 4);
#ifdef SB_EMU_TRACE
        if (lane == 0) fprintf(stderr, "serial copy base=%u cand=%u len=%u\n", base, cand, end - base);
#endif
        k1_push(ring, head, k1_event(base, end - base, base - cand));
        k1_preinsert(win, table, shift, s_limit, end);
        st.s = end; st.rematch = true;
        if (st.s >= target) return false;
    }
}

// A step covers the 64 positions [w, w + 64) with w = s & ~31: lane l owns position w + l (half 0) and w + 32 + l
// (half 1). The sequential words a lane needs for one half, fetched one step ahead when the block lives in global
// memory (hides one L2 round trip per step)
struct K1Seq { uint32_t a0, a1, a2, a3, a4, w; };
SB_DEVICE K1Seq k1_fetch_seq(const uint8_t* win, uint32_t w, uint32_t n) {
    const uintptr_t aa = (uintptr_t)(win + w + lane_id());
    const uint32_t* aw = (const uint32_t*)(aa & ~(uintptr_t)3);
#ifdef SB_EMU
    if (any((const uint8_t*)(aw + 5) > win + n)) K1_COUNT(3);   // a word reaches byte n or beyond (must stay 0)
#else
    (void)n;
#endif
    K1Seq q;
    q.a0 = aw[0]; q.a1 = aw[1]; q.a2 = aw[2]; q.a3 = aw[3]; q.a4 = aw[4]; q.w = w;
    return q;
}

// A half's probe between its issue and its use: the lane's hash, the table slot and the
// candidate's five aligned words, whose loads may still be in flight.
struct K1Probe { uint32_t h, c, b0, b1, b2, b3, b4; };
SB_DEVICE K1Probe k1_probe_issue(const uint8_t* win, const uint16_t* table, unsigned shift, const K1Seq& q) {
    const unsigned ash = (unsigned)((uintptr_t)(win + q.w + lane_id()) & 3u) * 8;
    K1Probe r;
    r.h = K1_HASH(funnel_r(q.a0, q.a1, ash));
    r.c = table[r.h];
    const uint32_t* bw = (const uint32_t*)((uintptr_t)(win + r.c) & ~(uintptr_t)3);
    r.b0 = bw[0]; r.b1 = bw[1]; r.b2 = bw[2]; r.b3 = bw[3]; r.b4 = bw[4];
    return r;
}

// one position probed against the table as it was when the probe was issued
struct K1Hit {
    uint32_t h;      // hash of the position
    uint32_t c;      // candidate read from the table
    uint32_t L;      // match length: exact up to 15, 16 = "16 or more"
    bool eq;         // a probe here would hit
};
SB_DEVICE K1Hit k1_probe_match(const uint8_t* win, const K1Seq& q, const K1Probe& pb) {
    const unsigned ash = (unsigned)((uintptr_t)(win + q.w + lane_id()) & 3u) * 8;
    const uint32_t a0 = q.a0, a1 = q.a1, a2 = q.a2, a3 = q.a3, a4 = q.a4;
    const uint32_t b0 = pb.b0, b1 = pb.b1, b2 = pb.b2, b3 = pb.b3, b4 = pb.b4;
    const unsigned bsh = (unsigned)((uintptr_t)(win + pb.c) & 3u) * 8;
    K1Hit r;
    r.h = pb.h;
    r.c = pb.c;
    r.eq = funnel_r(a0, a1, ash) == funnel_r(b0, b1, bsh);
    // match length, branch-free: bytes 4..15 of both sides, first differing byte wins
    {
        const uint32_t x4 = funnel_r(a1, a2, ash) ^ funnel_r(b1, b2, bsh);
        const uint32_t x8 = funnel_r(a2, a3, ash) ^ funnel_r(b2, b3, bsh);
        const uint32_t x12 = funnel_r(a3, a4, ash) ^ funnel_r(b3, b4, bsh);
        // the first word that differs and its base are selected first: one find-first-set instead of three
        const uint32_t x = x4 ? x4 : x8 ? x8 : x12;
        const uint32_t lb = x4 ? 4u : x8 ? 8u : 12u;
        r.L = x ? lb + ((uint32_t)(ffs(x) - 1) >> 3) : 16;
    }
    return r;
}

// "Next copy start" pointer doubling over the step's 64 positions. Node x's successor is the first hit at or after
// the end x + L of its copy (a rematch hit at the end itself, else the first later hit of the scan), 64 for none.
// Successors lie after their node, so a half-1 node's chain stays in half 1: each half doubles on its own, and a
// half-0 chain records where it leaves half 0. Copies are >= 4 bytes long and do not overlap, so a chain holds at most
// 8 copy starts in a half: three rounds (2^3 nodes) always reach its end.
struct K1Chains {
    uint32_t M0;     // half-0 copy starts reachable from the lane's half-0 node
    uint32_t X0;     // first node at or past 32 that chain reaches (64: none)
    uint32_t M1;     // half-1 copy starts reachable from the lane's half-1 node (bit i: position 32 + i)
    uint32_t bad;    // ballot: after the copy of the half-0 node, the scan leaves stride 1 inside the step
};
SB_DEVICE K1Chains k1_double(uint64_t E, bool eq0, uint32_t L0, bool eq1, uint32_t L1) {
    const unsigned lane = lane_id();
    const uint32_t e0 = lane + L0, e1 = 32 + lane + L1;
    uint32_t T0 = 64, T1 = 64;
    if (eq0 && e0 < 64) { const uint64_t m = E >> e0; if (m) T0 = e0 + (uint32_t)(ffsll(m) - 1); }
    if (eq1 && e1 < 64) { const uint64_t m = E >> e1; if (m) T1 = e1 + (uint32_t)(ffsll(m) - 1); }
    K1Chains r;
    // a rematch miss at e0 starts a scan at e0 + 1 with skip 32; it probes up to the next copy start or the end of
    // the step, and more than 32 such probes would leave stride 1 (a half-1 copy ends at 36 or later: never)
    r.bad = ballot(eq0 && (T0 < 64 ? T0 : 63u) > e0 + 32);
    uint32_t M0 = 1u << lane, M1 = 1u << lane;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint32_t M0n = shfl(M0, T0 & 31u), T0n = shfl(T0, T0 & 31u);
        const uint32_t M1n = shfl(M1, T1 & 31u), T1n = shfl(T1, T1 & 31u);
        if (T0 < 32) { M0 |= M0n; T0 = T0n; }
        if (T1 < 64) { M1 |= M1n; T1 = T1n; }
    }
    r.M0 = M0; r.X0 = T0; r.M1 = M1;
    return r;
}

// a step's two halves after the compare: hits, hit ballots over the 64 positions and the doubled chains
struct K1Pre {
    K1Hit x0, x1;
    uint64_t E;      // a probe at position i would hit
    uint64_t longs;  // hit whose length is only known to be >= 16
    K1Chains ch;
};
SB_DEVICE K1Pre k1_probe_complete(const uint8_t* win, const K1Seq* q, const K1Probe* pb) {
    K1Pre r;
    r.x0 = k1_probe_match(win, q[0], pb[0]);
    r.x1 = k1_probe_match(win, q[1], pb[1]);
    r.E = ballot(r.x0.eq) | (uint64_t)ballot(r.x1.eq) << 32;
    r.longs = ballot(r.x0.eq && r.x0.L == 16) | (uint64_t)ballot(r.x1.eq && r.x1.L == 16) << 32;
    r.ch = k1_double(r.E, r.x0.eq, r.x0.L, r.x1.eq, r.x1.L);
    return r;
}

// positions [x + 1, x + L - 2] of a copy at x (L >= 4), clipped to the step: not inserted; branch-free
SB_DEVICE uint64_t k1_interior(uint32_t x, uint32_t L) {
    const uint32_t hi = x + L - 2;
    const uint64_t upto = hi >= 63 ? ~0ull : ((2ull << hi) - 1ull);
    return upto & ~((2ull << x) - 1ull);                          // (2 << 63) wraps to 0: position 63 has no interior
}

// the step's copies to the ring in position order; slot0 / slot1: a lane's event among them for each half
SB_DEVICE void k1_push_copies(const K1Ring& r, K1Prod& pr, uint32_t ncopy, bool taken0, uint32_t slot0, uint64_t ev0,
                              bool taken1, uint32_t slot1, uint64_t ev1) {
    if (!ncopy) return;
    k1_wait_space(r, pr, ncopy);
    if (taken0) r.ev[(pr.head + slot0) & (r.size - 1)] = ev0;
    if (taken1) r.ev[(pr.head + slot1) & (r.size - 1)] = ev1;
    pr.head += ncopy;
    if (pr.head - pr.published >= K1_PUBLISH) k1_publish(r, pr);
}

// Finish one step from a probe result that is known to be current for every lane
// from the entry position on. Returns false (state untouched, table restored) when
// the step must be replayed serially. `nxt` holds the sequential words prefetched for w + 64 and w + 96;
// `hoisted` tells whether the next step's probe was issued into `nextp` (DESIGN.md section 4).
SB_DEVICE bool k1_finish(const uint8_t* win, uint32_t n, uint16_t* table, unsigned shift, uint32_t s_limit,
                         K1State& st, const K1Ring& ring, K1Prod& head, const K1Pre& pre, const K1Seq* nxt,
                         K1Probe* nextp, bool& hoisted K1_PROF_ARGS) {
    const unsigned lane = lane_id();
    hoisted = false;
    const uint32_t w = st.s & ~31u, i0 = st.s - w, p0 = w + lane, p1 = p0 + 32;
    const uint32_t h0 = pre.x0.h, c0 = pre.x0.c, h1 = pre.x1.h, c1 = pre.x1.c;
    const uint64_t E = pre.E;
    uint32_t L0 = pre.x0.L, L1 = pre.x1.L;
    // first copy start from the entry state: a rematch probe at i0 or a scan from i0, i.e. the first hit at/after i0
    const uint64_t fm = E >> i0;                                 // i0 < 32
    const uint32_t f = fm ? i0 + (uint32_t)(ffsll(fm) - 1) : 64;
    // the scan up to it (or to the end of the step) stays at stride 1: after a rematch miss at i0 it probes i0 + 1..f
    // with skip from 32, else i0..f with the running skip
    if ((st.rematch ? 31u : st.skip) + (f < 64 ? f : 63u) - i0 >= 64) return false;
    // ---- which hits are taken: the probe's pointer doubling, redone only when a taken copy's length is not exact
    // yet (>= 16) and its end can fall inside the step: that copy is extended cooperatively first
    uint64_t longmask = pre.longs;
    K1Chains ch = pre.ch;
    uint32_t CS0, CS1;                                           // taken copy starts: positions i, 32 + i
    for (;;) {
        const uint32_t fs = f & 31u;
        const uint32_t X0 = shfl(ch.X0, fs), M0 = shfl(ch.M0, fs);
        const uint32_t X = f < 32 ? X0 : f;                      // the entry chain's first node in half 1
        CS0 = f < 32 ? M0 : 0u;
        CS1 = X < 64 ? shfl(ch.M1, X & 31u) : 0u;
        const uint64_t unk = (CS0 | (uint64_t)CS1 << 32) & longmask;
        if (!unk) break;
        const unsigned j = ffsll(unk) - 1;
        const uint32_t pj = w + j, cj = shfl(j < 32 ? c0 : c1, j & 31u);
        const uint32_t end = k1_extend(win, n, pj + 16, cj + 16);
        if (lane == (j & 31u)) { if (j < 32) L0 = end - pj; else L1 = end - pj; }
        longmask &= ~(1ull << j);
        // a copy from 48 on ends past the step whatever its length: its node keeps "no successor"
        if (j < 48) ch = k1_double(E, pre.x0.eq, L0, pre.x1.eq, L1);
    }
    if (CS0 & ch.bad) return false;                              // a scan after a taken copy leaves stride 1
    K1_TICK(3);                                                  // [3] entry state -> taken copies (+ long extensions)
    // ---- inserted positions = entry..63 minus copy interiors [q+1, e-2]
    const bool taken0 = (CS0 >> lane) & 1u, taken1 = (CS1 >> lane) & 1u;
    const uint64_t interior = (taken0 ? k1_interior(lane, L0) : 0ull) | (taken1 ? k1_interior(32 + lane, L1) : 0ull);
    const uint32_t C0 = (0xFFFFFFFFu << i0) & ~reduce_or((uint32_t)interior);
    const uint32_t C1 = ~reduce_or((uint32_t)(interior >> 32));
    const bool ins0 = (C0 >> lane) & 1u, ins1 = (C1 >> lane) & 1u;
#ifdef SB_EMU_TRACE
    if (lane == 0) fprintf(stderr, "step w=%u i0=%u rm=%d skip=%u E=%016llx f=%u CS=%08x%08x C=%08x%08x\n", w, i0,
                           (int)st.rematch, st.skip, (unsigned long long)E, f, CS1, CS0, C1, C0);
#endif
    K1_TICK(4);                                                  // [4] interiors / inserted mask
    // the last writer of a slot wins: half 1 is stored after half 0, and within a half exactly one store lands
    // (detected below)
    syncwarp();                                                  // every lane's probe read precedes the commit
    if (ins0) table[h0] = (uint16_t)p0;
    syncwarp();
    if (ins1) table[h1] = (uint16_t)p1;
    syncwarp();
    const bool clash = (ins0 && table[h0] != (uint16_t)p0) | (ins1 && table[h1] != (uint16_t)p1);
    const uint32_t below = (1u << lane) - 1u, above = ~((2u << lane) - 1u);
    if (any(clash)) {
        // Two inserted positions share a slot. A probed position with an earlier inserted position of the same
        // slot should have seen that one as its candidate ("victim"): everything before the first victim is still
        // exactly what the serial encoder does, so keep that prefix and restart the step at the victim. Copy-end
        // pre-inserts (e-1) are write-only, never victims. Pairs within a half are found with match.any; a half-1
        // position whose slot holds a half-0 one is found by re-reading the table with only half 0 committed.
        const uint32_t same0 = match_any(ins0 ? h0 : 0xFFFF0000u | lane);
        const uint32_t same1 = match_any(ins1 ? h1 : 0xFFFF0000u | lane);
        uint64_t pre_bit = 0;
        if (taken0 && lane + L0 - 1 < 64) pre_bit |= 1ull << (lane + L0 - 1);
        if (taken1 && lane + L1 - 1 < 32) pre_bit |= 1ull << (32 + lane + L1 - 1);
        const uint32_t PRE0 = reduce_or((uint32_t)pre_bit), PRE1 = reduce_or((uint32_t)(pre_bit >> 32));
        // restore (same-slot lanes restore the same value), then commit the accepted prefix of half 0 with "highest
        // position of a slot wins"
        syncwarp();
        if (ins0) table[h0] = (uint16_t)c0;
        if (ins1) table[h1] = (uint16_t)c1;
        syncwarp();
        const uint32_t v0 = ballot(ins0 && !((PRE0 >> lane) & 1u) && (same0 & C0 & below) != 0);
        uint32_t cut = v0 ? ffs(v0) - 1 : 64;                    // step accepted up to (not including) this position
        const uint32_t keep0 = C0 & (cut >= 32 ? 0xFFFFFFFFu : ((1u << cut) - 1u));
        if (((keep0 >> lane) & 1u) && (same0 & keep0 & above) == 0) table[h0] = (uint16_t)p0;
        syncwarp();
        if (cut == 64) {
            // half 0 is committed whole: a half-1 slot that no longer holds its candidate holds a half-0 position
            const bool cross = ins1 && table[h1] != (uint16_t)c1;
            const uint32_t v1 = ballot(ins1 && !((PRE1 >> lane) & 1u) && (cross || (same1 & C1 & below) != 0));
            if (v1) cut = 32 + ffs(v1) - 1;
            const uint32_t keep1 = C1 & (cut >= 64 ? 0xFFFFFFFFu : ((1u << (cut - 32)) - 1u));
            syncwarp();
            if (((keep1 >> lane) & 1u) && (same1 & keep1 & above) == 0) table[h1] = (uint16_t)p1;
            syncwarp();
        }
        if (cut < 64) {
            if (cut < 32) { CS0 &= (1u << cut) - 1u; CS1 = 0; }
            else CS1 &= (1u << (cut - 32)) - 1u;
            const bool t0 = (CS0 >> lane) & 1u, t1 = (CS1 >> lane) & 1u;
            const uint32_t n0 = popc(CS0), ncut = n0 + popc(CS1);
            k1_push_copies(ring, head, ncut, t0, popc(CS0 & below), k1_event(p0, L0, p0 - c0),
                           t1, n0 + popc(CS1 & below), k1_event(p1, L1, p1 - c1));
            if (ncut) {
                const uint32_t e2 = reduce_max(t1 ? 32 + lane + L1 : t0 ? lane + L0 : 0u);   // <= cut: the victim is not inside a copy
                if (e2 == cut) { st.s = w + cut; st.rematch = true; }
                else { st.s = w + cut; st.rematch = false; st.skip = 32 + (cut - e2 - 1); }
            } else {
                st.skip = st.rematch ? 32 + (cut - i0 - 1) : st.skip + (cut - i0);
                st.s = w + cut; st.rematch = false;
            }
            return true;
        }
    }
    K1_TICK(5);                                                  // [5] commit + verify (+ clash handling)
    // ---- exit state and copy-end insert
    // (warp-uniform values, written as selects: only the copy-end insert below is a branch)
    const uint32_t n0 = popc(CS0), ncopy = n0 + popc(CS1);
    // the end of the lane's last copy: its half-1 one when taken (a taken half-0 copy that reaches 32 + lane covers it)
    const uint32_t e_mine = taken1 ? 32 + lane + L1 : taken0 ? lane + L0 : 0u;
    // hash of the word at e - 1 for a copy ending at e in 65..96 (the copy-end insert below), fetched by every lane for
    // its own copy end while the reduction that finds the last copy runs, instead of by index after it
    const unsigned nsh = (unsigned)((uintptr_t)(win + nxt[0].w + lane) & 3u) * 8;
    const uint32_t hend = shfl(K1_HASH(funnel_r(nxt[0].a0, nxt[0].a1, nsh)), (e_mine - 65) & 31u);
    const uint32_t e_last = reduce_max(e_mine);                  // end of the step's last copy, 0 without one
    const bool over = e_last >= 64;                              // that copy ends at or beyond the step's end
    // else the step ends in a scan: probes since the last copy end, since the rematch miss at i0, or the running scan's
    const uint32_t scan_skip = (CS0 | CS1) ? 32 + (63 - e_last) : st.rematch ? 32 + (63 - i0) : st.skip + (64 - i0);
    st.s = w + (over ? e_last : 64);
    st.skip = over ? st.skip : scan_skip;
    st.rematch = over;
    if (e_last >= 65) {                                          // e-1 lies beyond this step
        if (nxt[0].w == w + 64 && e_last <= 96) {
            // ... but inside the next step's first half, whose sequential words are already prefetched: take
            // its hash from the lane that holds it instead of paying a global load (:293-295)
            if (st.s < s_limit) {
                syncwarp();
                if (e_mine == e_last) table[hend] = (uint16_t)(st.s - 1);   // the last copy's lane
                syncwarp();
            }
        } else {
            k1_preinsert(win, table, shift, s_limit, st.s);
        }
    }
    const uint32_t slot0 = popc(CS0 & below), slot1 = n0 + popc(CS1 & below);   // this lane's events among the step's
    K1_TICK(7);                                                  // [7] exit state / copy-end insert
    // ---- the next step's probe. Every table store of this step is done, so when the next step is w + 64 on the
    // fast path its probe reads exactly the table it would read later: issue it now so that its candidate loads
    // overlap the ring stores and the next step's prefetch (k1_parse keeps such steps in its inner loop)
    hoisted = nxt[0].w == w + 64 && (st.s & ~31u) == w + 64 && k1_fast(w + 64, st, s_limit);
    if (hoisted) {
        nextp[0] = k1_probe_issue(win, table, shift, nxt[0]);
        nextp[1] = k1_probe_issue(win, table, shift, nxt[1]);
    }
    // ---- publish the copies
    k1_push_copies(ring, head, ncopy, taken0, slot0, k1_event(p0, L0, p0 - c0), taken1, slot1, k1_event(p1, L1, p1 - c1));
    K1_TICK(6);                                                  // [6] probe issue + event ring
    return true;
}

// Parser warp: block visible through `win` (global memory), n >= 17. One 64-position step at a time;
// the sequential words of the next step are requested before the current one is probed.
//   ctrl[6..7] = ring producer counters (head, published), carried from unit to unit
SB_DEVICE void k1_parse(const uint8_t* win, uint32_t n, uint16_t* table, const K1Ring& ring, uint32_t* ctrl) {
    const unsigned lane = lane_id();
    unsigned shift = 24;
    uint32_t tsize = 256;
    while (tsize < 16384 && tsize < n) { shift--; tsize *= 2; }   // src/compress.rs:491-497
    const uint32_t s_limit = n - 15;
    K1Prod prod;
    prod.head = ld_volatile(&ctrl[6]); prod.published = ld_volatile(&ctrl[7]); prod.tail_seen = 0;
    K1Seq seq[2];
    seq[0].a0 = seq[0].a1 = seq[0].a2 = seq[0].a3 = seq[0].a4 = 0; seq[0].w = 0xFFFFFFFFu;
    seq[1] = seq[0];
    K1_PROF_DECL
    K1State st;
    st.s = 1; st.skip = 32; st.rematch = false;
    for (;;) {
        uint32_t w = st.s & ~31u;
        bool finished;
        // fast-path test first: when it holds (w + 68 < s_limit, stride 1) neither end-of-block test can
        const bool fast = k1_fast(w, st, s_limit);
        if (!fast && (st.rematch ? st.s >= s_limit : st.s + (st.skip >> 5) > s_limit)) finished = true;
        else {
            bool ok = false;
            if (fast) {
                // the next step's words, when a step at w + 64 can run on the fast path: issue their loads now
                K1Seq nxt[2] = {seq[0], seq[1]};
                if (w + 64 + 68 < s_limit) { nxt[0] = k1_fetch_seq(win, w + 64, n); nxt[1] = k1_fetch_seq(win, w + 96, n); }
                K1_TICK(0);                                          // [0] loop top / state checks / prefetch issue
                K1Seq cur[2];
                cur[0] = seq[0].w == w ? seq[0] : k1_fetch_seq(win, w, n);
                cur[1] = seq[1].w == w + 32 ? seq[1] : k1_fetch_seq(win, w + 32, n);
                K1Probe pb[2];
                pb[0] = k1_probe_issue(win, table, shift, cur[0]);
                pb[1] = k1_probe_issue(win, table, shift, cur[1]);
                K1_COUNT(1);
                // While a step issues its successor's probe (`hoisted`), the successor runs in this inner loop
                // and not from the loop top: there the compiler joins all paths of the parse and waits for every
                // load in flight, which would put the candidate loads back on the critical path. For the same
                // reason the successor's own prefetch is issued only after its candidates are compared.
                K1_TICK(11);                                         // [11] probe issue (loop top)
#ifdef SB_EMU
                if (any(table[pb[0].h] != (uint16_t)pb[0].c || table[pb[1].h] != (uint16_t)pb[1].c)) K1_COUNT(2);
#endif
                K1Pre pre = k1_probe_complete(win, cur, pb);
                K1_TICK(1);                                          // [1] candidate wait, compare, doubling
                for (;;) {
                    seq[0] = nxt[0]; seq[1] = nxt[1];
                    bool hoisted;
                    ok = k1_finish(win, n, table, shift, s_limit, st, ring, prod, pre, seq, pb, hoisted K1_PROF_PASS);
                    if (!hoisted) break;
                    w += 64;                                         // == st.s & ~31u, on the fast path
                    cur[0] = seq[0]; cur[1] = seq[1];
                    K1_TICK(0);
                    K1_COUNT(0);
#ifdef SB_EMU
                    if (any(table[pb[0].h] != (uint16_t)pb[0].c || table[pb[1].h] != (uint16_t)pb[1].c)) K1_COUNT(2);
#endif
                    pre = k1_probe_complete(win, cur, pb);
                    K1_TICK(1);
                    // unconditional (this step's own words when w + 64 cannot be a fast step): a conditional load
                    // would become register moves that wait for it
                    const bool ahead = w + 64 + 68 < s_limit;
                    nxt[0] = k1_fetch_seq(win, ahead ? w + 64 : w, n);
                    nxt[1] = k1_fetch_seq(win, ahead ? w + 96 : w + 32, n);
                    // the words that the next step fetches come from HBM: have L2 fetch them now, so that the
                    // load finds them in L2 when its turn comes (a prefetch has no register to wait for)
                    prefetch_l2(win + (w + 160 + 2 * lane < n ? w + 160 + 2 * lane : n - 1));
                }
            }
            if (!ok) { K1_TICK(8); finished = k1_serial(win, n, table, shift, s_limit, st, w + 64, ring, prod); K1_TICK(9); }   // [9] serial path
            else finished = false;
        }
        if (finished) {
            k1_push(ring, prod, k1_event(n, 0, 0));                // end marker -> trailing literal (:417-426)
            k1_publish(ring, prod);
            K1_TICK(10);
            K1_PROF_FLUSH;
            syncwarp();
            if (lane == 0) { ctrl[6] = prod.head; ctrl[7] = prod.published; }
            return;
        }
    }
}
#undef K1_HASH

// ------------------------------------------------------------------- emitter
// Consumes copy events until the end marker (len == 0, pos == n); returns bytes written.
SB_DEVICE uint32_t k1_emit_block(const uint8_t* win, uint8_t* out, uint32_t d, const K1Ring& ring, uint32_t& tail) {
    const unsigned lane = lane_id();
    // output is write-once: evict-first stores keep it out of the L2 working set (windows + tables)
#define K1_OST(p, v) st8_stream((p), (uint8_t)(v))
#define K1_OCOPY warp_copy_t<true>
    uint32_t prev_end = 0;
    for (;;) {
        uint32_t avail;
        for (;;) {
            avail = ld_volatile(&ring.ctrl[0]) - tail;
            avail = shfl(avail, 0);
            if (avail) break;
            spin_long();
        }
        const uint32_t m = avail < 32 ? avail : 32;
        threadfence_block();                                  // every lane: the event loads below stay behind the head read
        uint64_t ev = 0;
        if (lane < m) ev = ld_volatile64(&ring.ev[(tail + lane) & (ring.size - 1)]);   // the ring may live in global memory
        const uint32_t pos = (uint32_t)(ev & 0x1FFFFu), len = (uint32_t)((ev >> 17) & 0x1FFFFu), off = (uint32_t)(ev >> 34);
        const bool act = lane < m;
        const bool is_end = act && len == 0;
        // literal in front of every event: [end of previous copy, pos)
        uint32_t pe = shfl_up(pos + len, 1);
        if (lane == 0) pe = prev_end;
        const uint32_t lit = act ? pos - pe : 0;
#ifdef SB_EMU_CHECK
        if (act && (pos < pe || pos > 65536)) fprintf(stderr, "BAD EVENT lane=%u m=%u tail=%u head_pub=%u pos=%u len=%u off=%u pe=%u prev_end=%u\n", lane, m, tail, ld_volatile(&ring.ctrl[0]), pos, len, off, pe, prev_end);
#endif
        uint32_t lhdr = 0;
        if (lit) lhdr = lit <= 60 ? 1 : lit <= 256 ? 2 : 3;                         // src/compress.rs:436-463
        // copy tags (src/compress.rs:339-356)
        uint32_t rem = len, n64 = 0, n60 = 0, fin = 0;
        if (act && len) {
            if (rem >= 68) { n64 = (rem - 68) / 64 + 1; rem -= 64 * n64; }
            if (rem > 64) { n60 = 1; rem -= 60; }
            fin = (rem <= 11 && off <= 2047) ? 2 : 3;
        }
        const uint32_t size = lhdr + lit + 3 * (n64 + n60) + fin;
        uint32_t incl = size;
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
            const uint32_t t = shfl_up(incl, k);
            if (lane >= (unsigned)k) incl += t;
        }
        uint8_t* o = out + d + (incl - size);
        if (lit) {
            const uint32_t mm = lit - 1;
            if (lhdr == 1) K1_OST(o, mm << 2);
            else if (lhdr == 2) { K1_OST(o, 60 << 2); K1_OST(o + 1, mm); }
            else { K1_OST(o, 61 << 2); K1_OST(o + 1, mm); K1_OST(o + 2, mm >> 8); }
            o += lhdr;
            if (lit <= 16) for (uint32_t k = 0; k < lit; k++) K1_OST(o + k, win[pe + k]);
        }
        // long literals: whole warp, one at a time
        uint32_t big = ballot(lit > 16);
        while (big) {
            const unsigned j = ffs(big) - 1;
            big &= big - 1;
            const uint32_t jl = shfl(lit, j), jp = shfl(pe, j);
            const uint32_t jo = shfl((uint32_t)(o - out), j);
            K1_OCOPY(out + jo, win + jp, jl);
        }
        if (act && len) {
            o += lit;
            for (uint32_t k = 0; k < n64; k++) { K1_OST(o, (63 << 2) | 2); K1_OST(o + 1, off); K1_OST(o + 2, off >> 8); o += 3; }
            if (n60) { K1_OST(o, (59 << 2) | 2); K1_OST(o + 1, off); K1_OST(o + 2, off >> 8); o += 3; }
            if (fin == 2) { K1_OST(o, ((off >> 8) << 5) | ((rem - 4) << 2) | 1); K1_OST(o + 1, off); }
            else { K1_OST(o, ((rem - 1) << 2) | 2); K1_OST(o + 1, off); K1_OST(o + 2, off >> 8); }
        }
        d += shfl(incl, 31);
        prev_end = shfl(pos + len, m - 1);
        tail += m;
        syncwarp();
        if (lane == 0) st_volatile(&ring.ctrl[1], tail);
        if (any(is_end)) return d;
    }
}


// One CTA per SM hosting NC + NG independent (parser, emitter) warp pairs. NC hash tables fill
// the SM's shared memory (7 x 32KB); NG further chains keep their table in an L2-resident global
// scratch (`gtables`, 32KB per chain): their probe/commit pays L2 latency, so each runs slower
// than a shared-memory chain, but they only use issue slots and registers the SM had idle.
// The window is read in place from global memory and the event rings live in an L2-resident
// global scratch (`ring_scratch`, K1_RING_GW entries per chain). Pairs synchronise on their own
// named barrier, so chains never wait for each other; because chains differ in speed they take
// units from a shared counter (`work`, zeroed by the host before the launch) instead of a
// fixed stride.
//   ctrl[8] = the unit this pair works on
// Unit limits (include/snapb200.h): a unit is one block, n <= 65536, and its output slot must hold
// max_compress_len(n) bytes; a unit that violates either is skipped with out_lens = 0 and, when the batch has a
// status array, TooBig / BufferTooSmall with the reference's payloads (src/compress.rs:104-117).
// The role is a template argument so that the parser's code does not keep the emitter's state (ring tail, output
// pointer) live across the parse: with one shared body the 7 + 5 and 7 + 7 kernels spill under their register caps.
template <bool parser>
SB_DEVICE void k1_chain(const BatchDesc& b, uint32_t flags, uint16_t* table, const K1Ring& ring, uint32_t* ctrl,
                        uint32_t* work, unsigned bar, uint32_t* crcs, const uint32_t* crc_tab) {
    const unsigned lane = lane_id();
    const unsigned pt = (parser ? 0u : 32u) + lane;                    // thread index within the pair
    uint32_t tail = 0;                // emitter's private ring counter (never reset)
    if (pt == 0) { ctrl[0] = 0; ctrl[1] = 0; ctrl[6] = 0; ctrl[7] = 0; }
    for (;;) {
        if (pt == 0) ctrl[8] = atomic_add(work, 1u);
        bar_sync(bar, 64);                                                 // previous unit fully drained, next one chosen
        const uint32_t u = ld_volatile(&ctrl[8]);
        if (u >= b.count) return;
        const uint8_t* in = unit_in(b, u);
        const uint32_t n = unit_in_len(b, u);
        uint8_t* out = unit_out(b, u);
        {
            const uint32_t cap = unit_out_cap(b, u), need = 32u + n + n / 6u;   // max_compress_len (:42-53)
            if (n > kMaxBlock || cap < need) {
                if (pt == 0) {
                    b.out_lens[u] = 0;
                    if (b.statuses) {
                        if (n > kMaxBlock) set_status(&b.statuses[u], SB_TOO_BIG, n, kMaxBlock, 0);
                        else set_status(&b.statuses[u], SB_BUFFER_TOO_SMALL, cap, need, 0);
                    }
                }
                bar_sync(bar, 64);
                continue;
            }
        }
        if (pt == 0 && b.statuses) set_status(&b.statuses[u], SB_OK, 0, 0, 0);
        uint32_t d = 0;
        if (flags & 1u) {                                                  // varint header (:120-128)
            uint32_t v = n;
            while (v >= 0x80) { if (pt == 0) out[d] = (uint8_t)v | 0x80; v >>= 7; d++; }
            if (pt == 0) out[d] = (uint8_t)v;
            d++;
        }
        if (n == 0) { if (pt == 0) { b.out_lens[u] = d; if (crcs) crcs[u] = 0; } bar_sync(bar, 64); continue; }
        {
            uint32_t tsize = 256;
            while (tsize < 16384 && tsize < n) tsize *= 2;
            if (tsize >= 512) for (uint32_t i = pt; i < tsize / 8; i += 64) ((uint4*)table)[i] = make_uint4(0, 0, 0, 0);   // (:514-516)
            else for (uint32_t i = pt; i < tsize / 2; i += 64) ((uint32_t*)table)[i] = 0;
        }
        bar_sync(bar, 64);
        if (parser) {
            if (n >= 17) k1_parse(in, n, table, ring, ctrl);           // (:140-150)
            else {                                                         // tiny block: one literal (:140-146)
                K1Prod prod;
                prod.head = ctrl[6]; prod.published = ctrl[7]; prod.tail_seen = 0;
                k1_push(ring, prod, k1_event(n, 0, 0));
                k1_publish(ring, prod);
                if (lane == 0) { ctrl[6] = prod.head; ctrl[7] = prod.published; }
            }
        } else {
            // frame encode: the chunk's masked CRC-32C is computed here, beside the compress call (src/frame.rs:76),
            // on issue slots the chain leaves idle while its parser produces the first events
            if (crcs) { const uint32_t crc = k3_warp_crc32c_masked1(crc_tab, in, n); if (lane == 0) crcs[u] = crc; }
            d = k1_emit_block(in, out, d, ring, tail);
            if (lane == 0) b.out_lens[u] = d;
        }
    }
}

// shared memory of a multi-chain CTA: NC tables + 64 control bytes per chain + the CRC byte table
constexpr size_t k1_multi_smem(int NC, int NG) { return (size_t)NC * K1_TABLE_BYTES + (size_t)(NC + NG) * 64 + K3_TABLE1_BYTES; }

template <int NC, int NG>
SB_DEVICE void k1_compress_body_multi(const BatchDesc& b, uint32_t flags, uint64_t* ring_scratch, uint16_t* gtables,
                                      uint32_t* work, uint32_t* crcs) {
    uint8_t* sm = smem();
    // Roles: with P chains in the CTA, warp c < P parses chain c and warp P + c emits for it. A warp is issued by the
    // scheduler (sub-partition) of its warp slot mod 4 and a CTA's warps take consecutive slots, so the parsers, which
    // bound the kernel, spread over all four schedulers (2/2/2/1 for P = 7). Pairing warps 2c / 2c + 1 would put every
    // parser on two schedulers and leave the other two to emitters that mostly sleep. A pair's named barrier does not
    // need its two warps to be adjacent.
    const unsigned P = block_dim() / 64, w = warp_id();
    const bool parser = w < P;
    const unsigned c = parser ? w : w - P;                             // chain within the CTA
    K1_PROF_CENSUS(parser);
    uint32_t* ctrl = (uint32_t*)(sm + (size_t)NC * K1_TABLE_BYTES + c * 64);
    uint32_t* crc_tab = (uint32_t*)(sm + (size_t)NC * K1_TABLE_BYTES + (size_t)(NC + NG) * 64);
    if (crcs) { k3_build_table1(crc_tab, thread_idx(), block_dim()); syncthreads(); }
    K1Ring ring;
    ring.size = K1_RING_GW;
    ring.ev = ring_scratch + ((size_t)block_idx() * (NC + NG) + c) * K1_RING_GW;
    ring.ctrl = ctrl;
    if (NG == 0 || c < NC) {
        uint16_t* table = (uint16_t*)(sm + (size_t)c * K1_TABLE_BYTES);
        if (parser) k1_chain<true>(b, flags, table, ring, ctrl, work, 1 + c, crcs, crc_tab);
        else k1_chain<false>(b, flags, table, ring, ctrl, work, 1 + c, crcs, crc_tab);
    } else {
        uint16_t* table = gtables + ((size_t)block_idx() * NG + (c - NC)) * (K1_TABLE_BYTES / 2);
        if (parser) k1_chain<true>(b, flags, table, ring, ctrl, work, 1 + c, crcs, crc_tab);
        else k1_chain<false>(b, flags, table, ring, ctrl, work, 1 + c, crcs, crc_tab);
    }
}

}  // namespace sbk

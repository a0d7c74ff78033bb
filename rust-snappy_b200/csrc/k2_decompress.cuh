// k2_decompress.cuh -- K2: batched raw Snappy decode, one stream per warp.
//
// Replaces reference src/decompress.rs:75-95 (Decoder::decompress), :130-148
// (element loop), :161-228 (read_literal), :233-343 (read_copy) and the tag
// table of build.rs:40-67, with the reference's exact error variants/payloads
// (src/error.rs:72-180) reported per stream.
//
// Design (not a port of the scalar loop): a warp looks at 32 consecutive
// compressed byte positions at once. Every lane decodes "the element that would
// start at my byte" speculatively, the true element boundaries are recovered by
// pointer doubling from lane 0 (which is always a true start), a warp scan of
// the output lengths gives every element its output position, literal payload
// bytes are scattered straight from the lanes that hold them, and copies are
// replayed in stream order with all lanes moving bytes. Errors are taken from
// the first true element in stream order that fails, so speculative lanes never
// raise errors the serial decoder would not reach.
#pragma once
#include "common.cuh"

namespace sbk {

static const uint32_t K2_SMEM_PER_WARP = 256;   // bytes of shared scratch per warp

// varint header: reference src/bytes.rs:73-90 + src/decompress.rs:362-374
// returns header length (0 = malformed) -- executed redundantly by all lanes.
SB_DEVICE uint32_t k2_read_header(const uint8_t* in, uint32_t n, uint64_t* value) {
    uint64_t v = 0;
    unsigned shift = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (shift >= 64) return 0;
        uint32_t b = in[i];
        if (b < 0x80) { *value = v | ((uint64_t)b << shift); return i + 1; }
        v |= (uint64_t)(b & 0x7F) << shift;
        shift += 7;
    }
    return 0;
}

// Decode one raw stream with the calling warp. Returns the status code. kHeader = false: `in` is the element sequence
// of one block alone (no varint header) that must produce exactly `cap` bytes -- K8 (k8_raw_split.cuh) hands every
// block of a split stream to its own warp this way, and the reference's checks are then made against the block's
// bounds, which are stricter than the stream's.
template <bool kHeader = true>
SB_DEVICE uint32_t k2_decode_stream(const uint8_t* in, uint32_t n, uint8_t* dst, uint64_t cap,
                                    sb_error* st, uint32_t* out_len, uint32_t* elems) {
    const unsigned lane = lane_id();
    uint64_t dn64 = cap;
    uint32_t hl = 0;
    if constexpr (kHeader) {
        if (n == 0) { if (lane == 0) set_status(st, SB_EMPTY, 0, 0, 0); return SB_EMPTY; }
        dn64 = 0;
        hl = k2_read_header(in, n, &dn64);
        if (hl == 0) { if (lane == 0) set_status(st, SB_HEADER, 0, 0, 0); return SB_HEADER; }
        if (dn64 > kMaxInput) { if (lane == 0) set_status(st, SB_TOO_BIG, dn64, kMaxInput, 0); return SB_TOO_BIG; }
        if (dn64 > cap) { if (lane == 0) set_status(st, SB_BUFFER_TOO_SMALL, cap, dn64, 0); return SB_BUFFER_TOO_SMALL; }
    }

    const uint8_t* src = in + hl;
    const uint8_t* in_end = in + n;
    const uint32_t sn = n - hl, dn = (uint32_t)dn64;        // both < 2^32 (checked above)
    uint32_t s = 0, d = 0;

    while (s < sn) {
#include "k2_window.inc"
        const bool is_start = ((M >> lane) & 1u) && valid;
        const unsigned last = 31 - clz(M);

        // ---- output position of every true element (spilling literal counts 0 here)
        uint32_t olen = (is_start && !spill) ? (uint32_t)len : 0u;
        uint32_t incl = olen;
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
            const uint32_t t = shfl_up(incl, k);
            if (lane >= (unsigned)k) incl += t;
        }
        const uint32_t opos = incl - olen;
        const uint32_t win_out = shfl(incl, 31);
        const uint64_t de = (uint64_t)d + opos;        // output position of my element
        const uint64_t sa = (uint64_t)s + lane + 1;    // stream position just after my tag byte

        // ---- errors. Cheap sufficient test first: 40 more input bytes (no truncated tag),
        // the whole window's output fits, no spilling literal, every copy offset is in range.
        // Only when that fails are the reference's checks evaluated element by element.
        const bool sure = (rem >= 40) && (dn - d >= win_out) &&
                          !any(is_start && (spill || (kind != 0 && (off == 0 || off > d + opos))));
        if (!sure) {
            // error conditions in the reference's order of checks
            uint32_t ecode = 0; uint64_t ea = 0, eb = 0, ec = 0;
            if (is_start) {
                if (kind == 0) {
                    uint64_t sp = sa;
                    if ((tag >> 2) >= 60) {
                        if (sa + 4 > sn) { ecode = SB_LITERAL; ea = 4; eb = sn - sa; ec = dn - de; }  // :192-198
                        sp = sa + (hdr - 1);
                    }
                    if (!ecode && (sn - sp < len || dn - de < len)) {                                   // :209-217
                        ecode = SB_LITERAL; ea = len; eb = sn - sp; ec = dn - de;
                    }
                } else {
                    const unsigned nb = hdr - 1;
                    if (sa + 4 > sn) {                                                                  // :439-472
                        if (nb == 1) { if (sa >= sn) { ecode = SB_COPY_READ; ea = 1; eb = sn - sa; } }
                        else if (nb == 2) { if (sa + 1 >= sn) { ecode = SB_COPY_READ; ea = 2; eb = sn - sa; } }
                        else { ecode = SB_COPY_READ; ea = 4; eb = sn - sa; }
                    }
                    if (!ecode && (off == 0 || de < off)) { ecode = SB_OFFSET; ea = off; eb = de; }     // :245-250
                    if (!ecode && de + len > dn) { ecode = SB_COPY_WRITE; ea = len; eb = dn - de; }     // :328-333
                }
            }
            const uint32_t emask = ballot(ecode != 0);
            if (emask) {
                const unsigned first = ffs(emask) - 1;
                if (lane == first) set_status(st, ecode, ea, eb, ec);
                return shfl(ecode, first);
            }
        }

        // ---- literal payload bytes that sit inside the window: lane -> output byte
        {
            const unsigned own = 31 - clz(M & (0xFFFFFFFFu >> (31 - lane)));  // nearest start <= lane
            const uint32_t pk = shfl((opos << 8) | (hdr << 4) | (kind << 1) | (spill ? 1u : 0u), own);
            const unsigned ohdr = (pk >> 4) & 0xFu;
            if (valid && (pk & 7u) == 0 && lane >= own + ohdr)
                dst[d + (pk >> 8) + (lane - own - ohdr)] = (uint8_t)tag;
        }
        syncwarp();

        // ---- copies. A copy whose source lies entirely before this window's output
        // (offset >= opos + len) depends on nothing written in this window. Those are flattened:
        // their bytes form one compact index space, one lane per copied byte, so a window's
        // ~30-60 copied bytes move in one or two warp-wide load/store pairs regardless of how many
        // copies they belong to. The rest (recent/overlapping sources, lengths above 32) are
        // replayed one by one in stream order afterwards.
        {
            uint8_t* const wout = dst + d;                       // window output base
            const uint32_t cpk = opos | ((uint32_t)len << 12);   // len <= 64 for copies, opos <= 2048
            const bool is_copy = is_start && kind != 0;
            const bool indep = is_copy && (uint32_t)len <= 32 && off >= opos + (uint32_t)len;
            const uint32_t im = ballot(indep);
            if (im) {
                // compact index of my first byte = prefix sum of independent copy lengths
                const uint32_t ilen = indep ? (uint32_t)len : 0u;
                uint32_t cincl = ilen;
#pragma unroll
                for (int k = 1; k < 32; k <<= 1) {
                    const uint32_t t2 = shfl_up(cincl, k);
                    if (lane >= (unsigned)k) cincl += t2;
                }
                const uint32_t cpos = cincl - ilen, ctot = shfl(cincl, 31);
                // element table in shared memory, indexed by rank among the independent copies
                if (indep) {
                    const uint32_t rk = popc(im & ((1u << lane) - 1u));
                    elems[rk * 2] = cpk | (cpos << 20);          // opos:12 | len:8 | cpos:12
                    elems[rk * 2 + 1] = off;
                }
                syncwarp();
                for (uint32_t base = 0; base < ctot; base += 64) {
                    uint32_t dsto[2], srco[2];
                    uint8_t v[2];
                    bool on[2];
#pragma unroll
                    for (int q = 0; q < 2; q++) {
                        const uint32_t lo = base + 32 * q;
                        // starts inside [lo, lo+32) -> bit; owner rank of byte t = starts at or before t, minus one
                        const uint32_t bit = (indep && cpos >= lo && cpos < lo + 32) ? 1u << (cpos - lo) : 0u;
                        const uint32_t Bm = reduce_or(bit);
                        const uint32_t before = popc(ballot(indep && cpos < lo));
                        const uint32_t t = lo + lane;
                        on[q] = t < ctot;
                        const uint32_t rk = before + popc(Bm & (0xFFFFFFFFu >> (31 - lane))) - 1;
                        const uint32_t e0 = on[q] ? elems[rk * 2] : 0u, e1 = on[q] ? elems[rk * 2 + 1] : 0u;
                        dsto[q] = (e0 & 0xFFFu) + (t - (e0 >> 20));
                        srco[q] = e1;
                    }
#pragma unroll
                    for (int q = 0; q < 2; q++) v[q] = on[q] ? wout[(int64_t)dsto[q] - (int64_t)srco[q]] : (uint8_t)0;   // offsets up to 2^32-1 are legal (:433-474)
#pragma unroll
                    for (int q = 0; q < 2; q++) if (on[q]) wout[dsto[q]] = v[q];
                }
            }
            syncwarp();
            uint32_t cm = ballot(is_copy && !indep);
            while (cm) {
                const unsigned j = ffs(cm) - 1;
                cm &= cm - 1;
                const uint32_t pk1 = shfl(cpk, j), coff = shfl(off, j);
                const uint32_t clen = pk1 >> 12;
                uint8_t* out = wout + (pk1 & 0xFFFu);
                if (coff >= clen || clen <= 32) {
                    // lanes below the offset read final bytes; an overlapping short copy is the
                    // periodic pattern of the last `coff` bytes (:306-317)
                    if (lane < clen) out[lane] = out[(int64_t)(coff >= clen || lane < coff ? lane : lane % coff) - (int64_t)coff];
                    if (clen > 32 && lane + 32 < clen) out[lane + 32] = out[(int64_t)lane + 32 - (int64_t)coff];
                } else {
                    const uint8_t* from = out - coff;
                    for (uint32_t k = lane; k < clen; k += 32) out[k] = from[k % coff];
                }
                syncwarp();
            }
        }

        // ---- window advance (+ the spilling literal, copied cooperatively)
        const uint32_t lpk = shfl((uint32_t)(spill ? 1u : 0u) | (hdr << 1), last);
        if (lpk & 1u) {
            const uint32_t llen = shfl((uint32_t)len, last);   // validated above: fits in 32 bits
            const uint32_t lsrc = s + last + (lpk >> 1);
            warp_copy(dst + d + win_out, src + lsrc, llen);
            syncwarp();
            s = lsrc + llen;
            d += win_out + llen;
        } else {
            s += shfl(E, 0);
            d += win_out;
        }
    }
    if (d != dn) {                                                                                   // :141-146
        if (lane == 0) set_status(st, SB_HEADER_MISMATCH, dn, d, 0);
        return SB_HEADER_MISMATCH;
    }
    if (lane == 0) { set_status(st, SB_OK, 0, 0, 0); if (out_len) *out_len = (uint32_t)dn; }
    return SB_OK;
}

// Kernel body: warp w of the grid decodes units w, w+nwarps, ...
SB_DEVICE void k2_decompress_body(const BatchDesc& b) {
    const unsigned warps_per_block = block_dim() >> 5;
    uint32_t* elems = (uint32_t*)smem() + warp_id() * 64;           // per-warp scratch: 32 x (packed element, offset)
    const uint64_t nwarps = (uint64_t)grid_dim() * warps_per_block;
    for (uint64_t u = (uint64_t)block_idx() * warps_per_block + warp_id(); u < b.count; u += nwarps) {
        const uint32_t i = (uint32_t)u;
        if (b.out_lens && lane_id() == 0) b.out_lens[i] = 0;
        k2_decode_stream(unit_in(b, i), unit_in_len(b, i), unit_out(b, i), unit_out_cap(b, i),
                         b.statuses ? &b.statuses[i] : nullptr, b.out_lens ? &b.out_lens[i] : nullptr, elems);
    }
}

}  // namespace sbk

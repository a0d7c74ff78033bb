/*
 * snapb200.h -- C ABI of the GPU-native (H100, sm_90a) Snappy codec (libsnapb200.so).
 *
 * This is the drop-in boundary for rust-snappy's raw/frame hot path: a Rust
 * `snap` shim (see INTEGRATION.md, rust/) binds exactly these symbols. Each
 * entry point cites the reference interface it replaces (paths relative to the
 * rust-snappy checkout). Plain pointers and sizes only -- no torch/CUDA types.
 *
 * All work is done by sm_90a CUDA kernels; there is NO CPU fallback. When no
 * CUDA device is usable every compute call returns SB_E_NO_DEVICE.
 */
#ifndef SNAPB200_H
#define SNAPB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* snap::Error variant index (declaration order of src/error.rs:72-180) plus
 * the payload fields of that variant in a, b, c. 0 = Ok. */
enum {
    SB_OK = 0,
    SB_TOO_BIG = 1,                  /* a=given  b=max                         */
    SB_BUFFER_TOO_SMALL = 2,         /* a=given  b=min                         */
    SB_EMPTY = 3,
    SB_HEADER = 4,
    SB_HEADER_MISMATCH = 5,          /* a=expected_len b=got_len               */
    SB_LITERAL = 6,                  /* a=len a=src_len c=dst_len              */
    SB_COPY_READ = 7,                /* a=len b=src_len                        */
    SB_COPY_WRITE = 8,               /* a=len b=dst_len                        */
    SB_OFFSET = 9,                   /* a=offset b=dst_pos                     */
    SB_STREAM_HEADER = 10,           /* a=byte                                 */
    SB_STREAM_HEADER_MISMATCH = 11,  /* a=6 body bytes, little endian          */
    SB_UNSUPPORTED_CHUNK_TYPE = 12,  /* a=byte                                 */
    SB_UNSUPPORTED_CHUNK_LENGTH = 13,/* a=len b=header(0/1)                    */
    SB_CHECKSUM = 14,                /* a=expected b=got                       */
    SB_IO_UNEXPECTED_EOF = 100,      /* io::ErrorKind::UnexpectedEof (read_exact, src/read.rs:439-455) */
    /* library-level failures (never produced by the reference) */
    SB_E_NO_DEVICE = 200,            /* no usable CUDA device / kernel image   */
    SB_E_CUDA = 201,                 /* a=cudaError_t                          */
    SB_E_INVALID = 202               /* bad argument (null pointer, ...)       */
};

typedef struct sb_error {
    uint32_t code;
    uint32_t _pad;
    uint64_t a, b, c;
} sb_error;

/* Outcome of a stream-ordered frame call, written to device memory by the last kernel of the call. */
typedef struct sb_frame_result {
    sb_error status;                 /* SB_OK or the first error in stream order                  */
    uint64_t bytes;                  /* encode: stream length; decode: bytes produced before the error */
    uint32_t nchunks;                /* data chunks in the stream                                  */
    uint32_t _pad;
} sb_frame_result;

/* ---- scalar API: host pointers, mirrors snap::raw ------------------------ */

/* snap::raw::max_compress_len  (src/compress.rs:42-53). Pure arithmetic. */
size_t sb_max_compress_len(size_t input_len);

/* snap::raw::Encoder::compress (src/compress.rs:99-154): `in` is compressed
 * as ONE raw stream (varint header + 64KB blocks) into out[..cap]; on success
 * returns 0 and *out_n = bytes written. Errors: TooBig, BufferTooSmall. */
int sb_compress(const uint8_t* in, size_t n, uint8_t* out, size_t cap, size_t* out_n, sb_error* err);

/* snap::raw::decompress_len (src/decompress.rs:30-35). Header parse only. */
int sb_decompress_len(const uint8_t* in, size_t n, size_t* out_len, sb_error* err);

/* snap::raw::Decoder::decompress (src/decompress.rs:75-95). Exact error
 * variant and payload of the reference on corrupt input. */
int sb_decompress(const uint8_t* in, size_t n, uint8_t* out, size_t cap, size_t* out_n, sb_error* err);

/* Stream-ordered raw decode of one stream d_in[0..n) in device memory into d_out[0..cap), caller scratch of
 * sb_decompress_scratch_bytes(n) bytes (sized from the compressed length alone), no allocation, no host
 * synchronisation. The stream's 64 KB blocks are located on the device and decoded in parallel, one warp per block;
 * a stream that is not split that way (copies reaching into an earlier block, elements across a block boundary,
 * literals over 64 KB, corrupt or truncated data) is decoded by one warp exactly as before. *d_result (device):
 * status = Ok or the reference's error, bytes = the decompressed length on Ok (0 otherwise), nchunks = blocks decoded
 * in parallel (0 when the one-warp path ran). On error d_out beyond what was decoded is unspecified. n above
 * 2^32 - 1, null pointers and scratch that is too small are SB_E_INVALID. sb_decompress takes this path for every
 * stream whose header announces more than 65536 bytes. */
uint64_t sb_decompress_scratch_bytes(uint64_t n);
int sb_decompress_device_ws(const uint8_t* d_in, uint64_t n, uint8_t* d_out, uint64_t cap,
                            sb_frame_result* d_result, void* scratch, uint64_t scratch_bytes,
                            void* stream, sb_error* err);

/* crc32::CheckSummer::crc32c_masked (src/crc32.rs:35-38), computed on device. */
int sb_crc32c_masked(const uint8_t* in, size_t n, uint32_t* out, sb_error* err);

/* ---- batched host API: many independent raw streams per call -------------
 * What a Rust caller holding many buffers (or the frame writers below) uses:
 * one call, pinned staging + H2D/D2H pipelined against the kernels inside.
 * Unit i reads in_base[in_offs[i] .. +in_lens[i]) and writes out_base[out_offs[i] ..];
 * out capacity per unit is out_caps[i]. statuses may be NULL for compress. A decode wave holding a unit whose
 * header announces more than 65536 bytes runs sb_decompress_batch_device_ws's block-parallel path. */
int sb_compress_batch_host(const uint8_t* in_base, const uint64_t* in_offs, const uint32_t* in_lens,
                           uint8_t* out_base, const uint64_t* out_offs, const uint32_t* out_caps,
                           uint32_t* out_lens, size_t count, sb_error* err);
int sb_decompress_batch_host(const uint8_t* in_base, const uint64_t* in_offs, const uint32_t* in_lens,
                             uint8_t* out_base, const uint64_t* out_offs, const uint32_t* out_caps,
                             uint32_t* out_lens, sb_error* statuses, size_t count, sb_error* err);
/* Same compress, but the LIBRARY lays the streams out back to back in out_base[0 .. out_cap) and reports where:
 * out_offs receives count+1 entries (out_offs[count] = total bytes). A caller cannot know compressed sizes in
 * advance, so this is the form whose drain is one D2H copy per wave; sb_max_compress_len(len) summed over the
 * units is always enough capacity. Units are one block each (in_lens[i] <= 65536, else TooBig). */
int sb_compress_batch_host_packed(const uint8_t* in_base, const uint64_t* in_offs, const uint32_t* in_lens,
                                  uint8_t* out_base, uint64_t out_cap, uint64_t* out_offs, uint32_t* out_lens,
                                  size_t count, sb_error* err);

/* ---- batched device API: device pointers, stream ordered ------------------
 * The kernels' native interface (and what bench.py's `value` times). All
 * pointers are device pointers; `stream` is a cudaStream_t passed as void*
 * (NULL is the legacy default stream, exactly as in the CUDA runtime).
 * Addressing is base + i*stride (uniform) -- or per-unit pointer arrays when
 * in_ptrs/out_ptrs are non-NULL. in_lens/out_caps NULL => the uniform value. */
typedef struct sb_batch {
    const uint8_t* const* in_ptrs;  const uint8_t* in_base;  uint64_t in_stride;
    const uint32_t* in_lens;        uint32_t in_len_uniform;
    uint8_t* const* out_ptrs;       uint8_t* out_base;       uint64_t out_stride;
    const uint32_t* out_caps;       uint32_t out_cap_uniform;
    uint32_t* out_lens;             /* device, count entries (required)      */
    sb_error* statuses;             /* device, count entries (decode; may be NULL for encode) */
    uint32_t count;
} sb_batch;

/* Each unit is ONE BLOCK: at most 65536 bytes, and its output slot must hold
 * sb_max_compress_len(len) bytes; the unit becomes one raw stream exactly as
 * Encoder::compress would produce it (one parser/emitter warp pair per unit, 12
 * pairs per SM). A unit that breaks either limit is skipped: out_lens[i] = 0 and,
 * when `statuses` is given, TooBig{given,max=65536} / BufferTooSmall{given,min}
 * (src/compress.rs:104-117); uniform lengths/caps are also checked on the host.
 * Larger inputs go through sb_compress / sb_frame_encode_device, which cut them
 * into blocks. Compress launches share a per-device scratch (event rings,
 * L2-resident hash tables, work counter): launches issued on different streams
 * of one device are ordered after each other on the device. */
int sb_compress_batch_device(const sb_batch* batch, void* stream, sb_error* err);
/* Each unit is one raw stream; statuses[i] carries the reference's error. */
int sb_decompress_batch_device(const sb_batch* batch, void* stream, sb_error* err);
/* The same per-unit results as sb_decompress_batch_device (bytes, out_lens[i], statuses[i] with the reference's
 * variant and payload; the same addressing), but every unit whose header announces more than 65536 bytes is split
 * into its 64 KB blocks as sb_decompress_device_ws splits one stream, and the blocks of all units are decoded side by
 * side in one grid. Units with at most one block, and units the split declines (a bad header or one over out_caps[i],
 * a header announcing more output than the compressed length can encode, copies into an earlier block, elements
 * across a block boundary, literals over 64 KB, corrupt or truncated data), are decoded by one warp exactly as before.
 *   in_bytes: the caller's upper bound on the sum of the units' in_lens (which may live on the device); the scratch,
 *     sb_decompress_batch_scratch_bytes(count, in_bytes) bytes, depends on nothing else. Bounds above 2^36 count as
 *     2^36. When the lengths sum to more than in_bytes, no unit is split: results stay exact.
 *   d_unit_blocks: optional (device, count entries): blocks decoded in parallel for unit i, 0 when one warp decoded it.
 * Stream ordered, no allocation, no host synchronisation. out_lens is required. Null pointers, count >= 2^31 and
 * scratch that is too small are SB_E_INVALID with nothing launched; count == 0 does nothing. */
uint64_t sb_decompress_batch_scratch_bytes(uint32_t count, uint64_t in_bytes);
int sb_decompress_batch_device_ws(const sb_batch* batch, uint64_t in_bytes, uint32_t* d_unit_blocks,
                                  void* scratch, uint64_t scratch_bytes, void* stream, sb_error* err);
/* Raw compress of units of ANY length: unit i becomes exactly what Encoder::compress(input_i, &mut output_i[..cap_i])
 * produces (src/compress.rs:99-154), cap_i = out_caps[i] or the uniform cap; the same addressing as the other batch
 * calls, and a uniform length over 65536 is legal. Every unit is cut into its 64 KB blocks and the blocks of all units
 * are compressed in one launch, then each unit's varint header and block bodies are assembled in its output. Per unit:
 *   Ok: out_lens[i] = the stream's length (an empty unit is the one byte 0x00).
 *   TooBig{given=n, max=2^32-1} when max_compress_len(n) == 0 (n > 3,681,400,511);
 *   BufferTooSmall{given=cap_i, min=max_compress_len(n)} when cap_i is smaller.
 *   A unit that is not compressed has out_lens[i] = 0 (every stream is at least one byte), and neither its input nor its
 *   output is touched. statuses may be NULL.
 *   in_bytes: the caller's bound on the sum of in_lens over units of MORE than 65536 bytes (0 for a batch of <= 64 KB
 *     units); the scratch, sb_compress_batch_scratch_bytes(count, in_bytes) bytes, depends on nothing else. When those
 *     lengths sum to more than in_bytes on the device, every such unit gets SB_E_INVALID{a=sum, b=in_bytes} and
 *     out_lens 0; units of at most 65536 bytes are still compressed. Rejected units do not count towards the sum.
 * Stream ordered, no allocation, no host synchronisation; with count 1 it is the device-resident sb_compress. Null
 * pointers (batch, out_lens, scratch), count >= 2^31, a bound whose block count does not fit one launch
 * (sb_compress_batch_scratch_bytes returns UINT64_MAX) and scratch that is too small are SB_E_INVALID with nothing
 * launched; count == 0 does nothing. Like sb_compress_batch_device, launches on different streams are ordered. */
uint64_t sb_compress_batch_scratch_bytes(uint32_t count, uint64_t in_bytes);
int sb_compress_batch_device_ws(const sb_batch* batch, uint64_t in_bytes, void* scratch, uint64_t scratch_bytes,
                                void* stream, sb_error* err);
/* Frame encode of units of ANY length: unit i becomes exactly what sb_frame_encode(input_i) produces, that is
 * `FrameEncoder::new(vec![]).write_all(input_i); into_inner()` (src/write.rs:123-192): the stream identifier, then one
 * chunk per <= 65536-byte slice, compressed or stored by the reference's rule. The same addressing as the other batch
 * calls; every chunk of every unit is compressed in one launch, then each unit is assembled in its output. Per unit, with
 * n = in_len_i and cap_i = out_caps[i] or the uniform cap:
 *   Ok: out_lens[i] = the stream's length; an empty unit writes nothing and has out_lens[i] = 0 (src/write.rs:155-157).
 *   BufferTooSmall{given=cap_i, min=sb_frame_max_len(n)} when cap_i is smaller (so every n > 3,679,453,184).
 *   A rejected unit has out_lens[i] = 0, and neither its input nor its output is touched. statuses may be NULL.
 *   in_bytes: as for sb_compress_batch_device_ws, the caller's bound on the sum of in_lens over units of MORE than 65536
 *     bytes; the scratch, sb_frame_encode_batch_scratch_bytes(count, in_bytes) bytes, depends on nothing else. When those
 *     lengths sum to more than in_bytes on the device, every such unit gets SB_E_INVALID{a=sum, b=in_bytes} and
 *     out_lens 0; units of at most 65536 bytes are still encoded.
 *   d_chunk_offs: optional (device). Unit i's index starts at entry i + sum_{j<i} ceil(n_j / 65536) and holds
 *     ceil(n_i / 65536) + 1 entries: the offset of every chunk header in the unit's output (the first is 10), then the
 *     stream length -- the index sb_frame_encode_device_ws emits and sb_frame_decode_device_ws accepts. An empty unit
 *     gets the single entry 0; a rejected unit's entries are not written.
 * Stream ordered, no allocation, no host synchronisation; a unit's input and output must not overlap. Null pointers
 * (batch, out_lens, scratch), count >= 2^31, a bound whose chunk count does not fit one launch
 * (sb_frame_encode_batch_scratch_bytes returns UINT64_MAX) and scratch that is too small are SB_E_INVALID with nothing
 * launched; count == 0 does nothing. Like sb_compress_batch_device, launches on different streams are ordered. */
uint64_t sb_frame_encode_batch_scratch_bytes(uint32_t count, uint64_t in_bytes);
int sb_frame_encode_batch_device_ws(const sb_batch* batch, uint64_t in_bytes, uint64_t* d_chunk_offs,
                                    void* scratch, uint64_t scratch_bytes, void* stream, sb_error* err);
/* Frame decode of a batch of streams: unit i is one frame stream, decoded as `FrameDecoder::new(unit_i).read_to_end()`
 * (src/read.rs:104-239). statuses[i] and out_lens[i] equal the status and bytes sb_frame_decode_device_ws(unit_i, cap_i,
 * ..., flags) writes to its sb_frame_result given a chunk table large enough, and out_i[0 .. out_lens[i]) equals that
 * call's output: Ok with the decoded length, the reader's first error in stream order with the bytes produced before
 * it, or BufferTooSmall{given=cap_i, min=decoded length} with nothing decoded. Beyond out_lens[i] a failing unit's
 * output is unspecified; an empty unit is Ok with 0 bytes. The same addressing as the other batch calls; statuses and
 * out_lens are required. Every unit's chunk index is built (or checked) in parallel and the chunks of all units are
 * decoded side by side in one grid; a unit that is not a clean run of data chunks is walked by one thread.
 *   flags bit0: no stream identifier expected, for every unit (fragments).
 *   d_chunk_offs, d_index_at: optional caller index (device), both or neither. Unit i's is
 *     d_chunk_offs[d_index_at[i] .. d_index_at[i+1]): the offset of every chunk header in the unit, then its length --
 *     the layout sb_frame_encode_batch_device_ws writes, where d_index_at[i] = i + sum_{j<i} ceil(n_j / 65536). An
 *     index that does not describe its unit costs speed, never a result: that unit is walked.
 *   in_bytes: the caller's bound on the sum of in_lens; it sizes only the parallel indexer's tables. When the lengths sum
 *     to more on the device, units without a caller index are walked: results stay exact. Bounds above 2^36 count as
 *     2^36.
 *   max_chunks: slots of the batch's chunk table, 1 .. 4,194,302. Units take ranges of data chunks in batch order; the
 *     first unit whose chunks do not fit and every unit after it get SB_E_INVALID{a=max_chunks, b=1} (the single call's
 *     "chunk table too small", with the same priority over BufferTooSmall) and out_lens 0. With a caller index the
 *     exact need is d_index_at[count] - d_index_at[0] - count; n_i / 8 summed over the units is always enough.
 *   d_unit_chunks: optional (device, count entries): the data chunks of unit i the parallel parse placed, 0 when one
 *     thread walked the unit.
 * Stream ordered, no allocation, no host synchronisation; the scratch, sb_frame_decode_batch_scratch_bytes(count,
 * in_bytes, max_chunks) bytes, depends on nothing else and need not be zeroed. Null pointers (batch, out_lens, statuses,
 * scratch), count >= 2^31, max_chunks == 0 or over the limit, an index given half and scratch that is too small are
 * SB_E_INVALID with nothing launched; count == 0 does nothing. */
uint64_t sb_frame_decode_batch_scratch_bytes(uint32_t count, uint64_t in_bytes, uint32_t max_chunks);
int sb_frame_decode_batch_device_ws(const sb_batch* batch, uint64_t in_bytes, uint32_t flags,
                                    const uint64_t* d_chunk_offs, const uint64_t* d_index_at, uint32_t max_chunks,
                                    uint32_t* d_unit_chunks, void* scratch, uint64_t scratch_bytes,
                                    void* stream, sb_error* err);
/* Masked CRC-32C of each unit (frame chunks): out_lens[i] receives the CRC. */
int sb_crc32c_masked_batch_device(const sb_batch* batch, void* stream, sb_error* err);

/* ---- frame format (snap::write::FrameEncoder / snap::read::FrameDecoder) --
 * One-shot forms over host memory. sb_frame_encode(in) produces exactly the
 * bytes of `FrameEncoder::new(vec![]).write_all(in); into_inner()`
 * (src/write.rs:123-192): stream identifier + one chunk per <=65536-byte slice;
 * empty input => empty output. */
size_t sb_frame_max_len(size_t n);
int sb_frame_encode(const uint8_t* in, size_t n, uint8_t* out, size_t cap, size_t* out_n, sb_error* err);
/* The chunk loop of write::Inner::write alone (src/write.rs:171-190): chunks for
 * `in` with (include_ident=1) or without the leading stream identifier -- what
 * a streaming FrameEncoder calls for every buffer it hands down. */
int sb_frame_encode_ex(const uint8_t* in, size_t n, uint8_t* out, size_t cap, size_t* out_n, int include_ident, sb_error* err);
/* `FrameDecoder::new(in).read_to_end()` (src/read.rs:104-239): pass out=NULL to
 * size the output (*out_n). Errors carry the reference's variant/payload. */
int sb_frame_decode(const uint8_t* in, size_t n, uint8_t* out, size_t cap, size_t* out_n, sb_error* err);

/* Device-resident frame encode of n bytes at d_in (device) into d_out (device,
 * cap >= sb_frame_max_len(n)); *out_n (host) = stream length. include_ident=0
 * omits the 10-byte stream identifier (ranks > 0 of a sharded stream).
 * Convenience form: pooled scratch, waits for the result. */
int sb_frame_encode_device(const uint8_t* d_in, uint64_t n, uint8_t* d_out, uint64_t cap,
                           int include_ident, uint64_t* out_n, void* stream, sb_error* err);

/* ---- stream-ordered frame calls with caller-provided scratch ---------------
 * No allocation, no host synchronisation (n > 0): every kernel of the call is
 * enqueued on `stream` and the outcome is written to *d_result (device memory).
 *   scratch: device memory of at least sb_frame_{encode,decode}_scratch_bytes(..).
 * Encode (src/write.rs:165-192 + src/frame.rs:62-104): K1 compresses every chunk
 * and leaves its masked CRC-32C beside it, a two-level scan places the chunks,
 * one gather writes headers + bodies. d_chunk_offs (optional, device, nchunks+1
 * entries) receives the offset of every chunk header in d_out and the total --
 * the chunk index sb_frame_decode_device_ws accepts. */
uint64_t sb_frame_encode_scratch_bytes(uint64_t n);
int sb_frame_encode_device_ws(const uint8_t* d_in, uint64_t n, uint8_t* d_out, uint64_t cap, int include_ident,
                              uint64_t* d_chunk_offs, sb_frame_result* d_result, void* scratch, uint64_t scratch_bytes,
                              void* stream, sb_error* err);
/* Decode (read::FrameDecoder, src/read.rs:104-239) of a frame stream in device
 * memory. With d_chunk_offs/nchunks (the encoder's index, or the one
 * sb_frame_index_device_ws builds; d_chunk_offs[nchunks] = n) the chunk headers
 * are parsed in parallel. Without it the decoder first builds the index itself
 * on the device (in its own scratch, no host synchronisation); when the stream is
 * not a clean run of data chunks (skippable/padding chunks, a repeated
 * identifier, ...) or an index does not describe it, one thread walks the
 * headers in stream order exactly like the reference's reader. Then one warp per chunk:
 * raw decode (K2) or copy, masked CRC-32C of the produced bytes against the
 * header. d_result: first error in stream order + bytes produced before it.
 *   flags bit0: no stream identifier expected (a rank's fragment of a sharded stream)
 *   max_chunks: capacity of the chunk table carved from scratch (SB_E_INVALID{a=max_chunks,b=1} if exceeded) */
uint64_t sb_frame_decode_scratch_bytes(uint32_t max_chunks);
int sb_frame_decode_device_ws(const uint8_t* d_in, uint64_t n, uint8_t* d_out, uint64_t cap,
                              const uint64_t* d_chunk_offs, uint32_t nchunks, uint32_t flags,
                              sb_frame_result* d_result, void* scratch, uint64_t scratch_bytes, uint32_t max_chunks,
                              void* stream, sb_error* err);
/* Convenience form: pooled scratch, waits and returns the result on the host. */
int sb_frame_decode_device(const uint8_t* d_in, uint64_t n, uint8_t* d_out, uint64_t cap,
                           const uint64_t* d_chunk_offs, uint32_t nchunks, uint32_t flags,
                           sb_frame_result* result, void* stream, sb_error* err);
/* Byte ranges of one frame stream in device memory: range r receives decoded bytes [d_lo[r], d_lo[r] + d_len[r]) in
 * d_out_ptrs[r] (device, d_len[r] bytes). Only the chunks a range covers are decoded and checksummed, so a window of a
 * stream far larger than device memory costs its own chunks and one pass over the headers. The index phase is
 * sb_frame_decode_device_ws's (d_chunk_offs/nchunks and flags bit0 work as there) and runs once per call.
 *   Ranges may be empty, unsorted, overlapping, duplicated, or reach past the end; output buffers must not overlap each
 *   other or the input. With end = min(lo + len, total), range r verifies chunk k (output offset off_k, decoded length
 *   dlen_k) iff off_k < end && off_k + max(dlen_k, 1) > lo: the chunks producing its bytes and the empty chunks inside
 *   it. Each verified chunk is decoded and its masked CRC-32C checked. d_statuses[r] and d_out_lens[r], in priority order:
 *     1. chunk table too small: SB_E_INVALID{a=max_chunks, b=1}, 0;
 *     2. a verified chunk fails: the first in stream order, k*, with its own status; max(off_k*, lo) - lo;
 *     3. the range reaches past total and the header walk stopped on an error: that error; max(end - lo, 0);
 *     4. otherwise Ok; max(end - lo, 0) (a range past a clean end is a short read, like pread).
 *   out[0 .. out_len) is exactly what FrameDecoder::new(stream).read_to_end() gives for those bytes when every chunk the
 *   range does not verify is valid; beyond it the bytes are unspecified. Nothing outside [out_r, out_r + max(end - lo,
 *   0)) is written, so a buffer may hold just the bytes the stream can give the range. For a stream
 *   sb_frame_decode_device_ws decodes Ok, every range is Ok and equals that output's slice.
 *   *d_result: the stream's walk status (Invalid{max_chunks, 1}, the walk's stopping error, or Ok), bytes = total (the
 *   decoded length of the chunks in the table) and nchunks. nranges == 0 writes only *d_result: the decoded length
 *   without decoding.
 *   max_chunks: chunk table slots, 1 .. 4,194,302.
 * A chunk shared by several ranges is decoded once per range, and the scratch,
 * sb_frame_decode_ranges_scratch_bytes(max_chunks, nranges) bytes, holds 128 KiB of staging per range for the chunks that
 * straddle a range's ends; split very many small ranges over several calls. Stream ordered, no allocation, no host
 * synchronisation, and the same number of launches whatever nranges. Null pointers that are needed, nranges >= 2^31,
 * max_chunks out of range, nchunks > max_chunks with an index and scratch that is too small are SB_E_INVALID with
 * nothing launched. */
uint64_t sb_frame_decode_ranges_scratch_bytes(uint32_t max_chunks, uint32_t nranges);
int sb_frame_decode_ranges_device_ws(const uint8_t* d_in, uint64_t n, const uint64_t* d_chunk_offs, uint32_t nchunks,
                                     uint32_t flags, const uint64_t* d_lo, const uint64_t* d_len, uint8_t* const* d_out_ptrs,
                                     uint64_t* d_out_lens, sb_error* d_statuses, uint32_t nranges, sb_frame_result* d_result,
                                     void* scratch, uint64_t scratch_bytes, uint32_t max_chunks, void* stream, sb_error* err);

/* Seek table of one frame stream in device memory, built on the device once and then read by
 * sb_frame_table_decode_ranges_device_ws any number of times without another pass over the stream's headers. The build
 * runs sb_frame_decode_ranges_device_ws's index phase (d_chunk_offs/nchunks, flags bit0 and max_chunks, 1 .. 4,194,302,
 * work as there) and writes the table to d_table, which must be 8-byte aligned and hold at least
 * sb_frame_table_bytes(max_chunks) bytes. *d_result is what sb_frame_decode_ranges_device_ws writes with nranges == 0: the
 * walk status, the decoded total and the chunk count.
 *   The table is a header (a magic word with the format version, the stream's compressed length n, the chunk count, the
 *   decoded total, the walk's stopping status, whether the chunk table was too small) and one 32-byte record per data
 *   chunk in stream order (body offset and length, decoded length, expected CRC, type, decoded offset). It holds no
 *   pointers, and its first sb_frame_table_bytes(result.nchunks) bytes are a complete table: it may be cut to that size,
 *   copied or moved. A walked stream (padding or skippable chunks, a repeated identifier) is walked here, once; its table
 *   lists only the data chunks.
 * Scratch: sb_frame_table_build_scratch_bytes(max_chunks). Stream ordered, no allocation, no host synchronisation, a fixed
 * number of launches. Null pointers, max_chunks out of range, nchunks > max_chunks with an index and a table or scratch
 * that is too small are SB_E_INVALID with nothing launched. */
uint64_t sb_frame_table_bytes(uint32_t nchunks);
uint64_t sb_frame_table_build_scratch_bytes(uint32_t max_chunks);
int sb_frame_table_build_device_ws(const uint8_t* d_in, uint64_t n, const uint64_t* d_chunk_offs, uint32_t nchunks,
                                   uint32_t flags, void* d_table, uint64_t table_bytes, uint32_t max_chunks,
                                   sb_frame_result* d_result, void* scratch, uint64_t scratch_bytes, void* stream,
                                   sb_error* err);
/* Seek tables of a batch of frame streams in one call, every unit indexed in parallel: what one
 * sb_frame_table_build_device_ws per stream gives, without a call per stream. Unit i is batch input i (in_ptrs or
 * in_base + stride, in_lens or the uniform length, count); the out_* fields, out_lens and statuses are not read. flags
 * bit0, d_chunk_offs/d_index_at (both or neither), in_bytes and max_chunks (1 .. 4,194,302) mean exactly what they mean
 * for sb_frame_decode_batch_device_ws: units take ranges of one chunk table of max_chunks slots in batch order, an index
 * that does not describe its unit costs speed, never a result, and lengths summing past in_bytes get units walked with
 * exact results.
 *   The tables are packed back to back in batch order into d_tables (device, 8-byte aligned, at least
 *   sb_frame_table_batch_bytes(count, max_chunks) = 64 * count + 32 * max_chunks bytes). d_table_offs (device, count + 1
 *   entries) gets d_table_offs[0] = 0 and d_table_offs[i + 1] = d_table_offs[i] + sb_frame_table_bytes(d_results[i].nchunks):
 *   every table size is a multiple of 32, so every table is 8-byte aligned, and the first d_table_offs[count] bytes may be
 *   kept with one copy.
 *   A unit that fits the chunk table gets a table and d_results[i] byte-identical (padding included) to the first
 *   sb_frame_table_bytes(nchunks) bytes of what sb_frame_table_build_device_ws writes for that stream alone with the same
 *   flags, its own index slice or none, and a max_chunks large enough: walked streams, fragments, corrupt chunks (a build
 *   checks no CRC), truncated streams and decoded totals over 2^32 alike. The first unit that does not fit and every unit
 *   after it get d_results[i] = {SB_E_INVALID{a=max_chunks, b=1}, 0, 0} and a 64-byte table (the stream's length, total 0,
 *   no chunks, chunk table too small, that status): every read of it gives that status and no bytes.
 * Scratch: sb_frame_table_build_batch_scratch_bytes(count, in_bytes, max_chunks), need not be zeroed. Stream ordered, no
 * allocation, no host synchronisation, and the same launches whatever count and the streams hold (one number with an
 * index, one without). Null pointers (batch, d_tables, d_table_offs, d_results, scratch), count >= 2^31, max_chunks out of
 * range, an index given half and tables or scratch that are too small are SB_E_INVALID with nothing launched; count == 0
 * does nothing. */
uint64_t sb_frame_table_batch_bytes(uint32_t count, uint32_t max_chunks);
uint64_t sb_frame_table_build_batch_scratch_bytes(uint32_t count, uint64_t in_bytes, uint32_t max_chunks);
int sb_frame_table_build_batch_device_ws(const sb_batch* batch, uint64_t in_bytes, uint32_t flags,
                                         const uint64_t* d_chunk_offs, const uint64_t* d_index_at, uint32_t max_chunks,
                                         void* d_tables, uint64_t tables_bytes, uint64_t* d_table_offs,
                                         sb_frame_result* d_results, void* scratch, uint64_t scratch_bytes, void* stream,
                                         sb_error* err);
/* Byte ranges of many tabled frame streams in one call. d_tables, d_ins and d_in_lens are device arrays of `count`
 * entries: stream u is d_ins[u][0 .. d_in_lens[u]) and d_tables[u] its seek table. Range r asks for decoded bytes
 * [d_lo[r], d_lo[r] + d_len[r]) of stream d_unit[r] into d_out_ptrs[r] (device, d_len[r] bytes). Ranges may be empty,
 * unsorted, overlapping, repeated, reach past the end and mix streams in any order; output buffers must not overlap each
 * other or the inputs. Only the chunks a range covers are decoded and checksummed. With total the table's decoded total
 * and end = min(lo + len, total), range r verifies chunk k (output offset off_k, decoded length dlen_k) iff
 * off_k < end && off_k + max(dlen_k, 1) > lo. d_statuses[r] and d_out_lens[r], in priority order:
 *   1. d_unit[r] >= count: SB_E_INVALID{a=unit, b=count, c=1}, 0;
 *   2. d_tables[u] is not a table of this format, or was built over a stream of another length than d_in_lens[u]:
 *      SB_E_INVALID{a=d_in_lens[u], b=the table's n (0 if it is not a table), c=2}, 0;
 *   3. the chunk table of the build was too small: SB_E_INVALID{a=max_chunks, b=1}, 0;
 *   4. a verified chunk fails: the first in stream order, k*, with its own status; max(off_k*, lo) - lo;
 *   5. the range reaches past total and the build's header walk stopped on an error: that error; max(end - lo, 0);
 *   6. otherwise Ok; max(end - lo, 0) (a range past a clean end is a short read, like pread).
 *   For a table built from stream S, every range gets exactly the status, out_len and bytes that
 *   sb_frame_decode_ranges_device_ws(S, ...) gives it with the same index, flags and max_chunks. Nothing outside
 *   [out_r, out_r + max(end - lo, 0)) is written.
 *   Tables are checked only as far as is cheap. Every decoded chunk is still CRC-checked, so a table paired with other
 *   bytes of the same length gives errors, not wrong output. A record a range uses must keep to the bounds every build
 *   writes (body inside the stream, body <= 76,490 bytes, decoded <= 65,536 bytes, a data chunk type, a non-negative
 *   slice of [lo, end)), else it fails as chunk k with SB_E_INVALID{a=k, b=0, c=3}; no table content makes the call read
 *   outside a stream or write outside a range's buffer or the scratch.
 * A chunk shared by several ranges is decoded once per range; the scratch, sb_frame_table_ranges_scratch_bytes(nranges)
 * bytes, holds 128 KiB of staging per range. Stream ordered, no allocation, no host synchronisation, and the same
 * launches whatever count and nranges; nranges == 0 does nothing. Null pointers that are needed, count or
 * nranges >= 2^31 and scratch that is too small are SB_E_INVALID with nothing launched. */
uint64_t sb_frame_table_ranges_scratch_bytes(uint32_t nranges);
int sb_frame_table_decode_ranges_device_ws(const void* const* d_tables, const uint8_t* const* d_ins,
                                           const uint64_t* d_in_lens, uint32_t count, const uint32_t* d_unit,
                                           const uint64_t* d_lo, const uint64_t* d_len, uint8_t* const* d_out_ptrs,
                                           uint64_t* d_out_lens, sb_error* d_statuses, uint32_t nranges, void* scratch,
                                           uint64_t scratch_bytes, void* stream, sb_error* err);

/* Seek tables of a batch of raw streams in one call, built from the 64 KiB block starts that
 * sb_decompress_batch_device_ws finds, every block decoded and checksummed once. Unit i is batch input i (in_ptrs or
 * in_base + stride, in_lens or the uniform length, count); the out_* fields, out_lens and statuses are not read. in_bytes
 * means what it means for sb_decompress_batch_device_ws.
 *   A raw table is a 64-byte header (a magic word with the format version, distinct from a frame table's; the stream's
 *   compressed length n; the varint header length hl; the decoded length dn; the block count ceil(dn / 65536); a
 *   seekable flag; the reason a stream is not seekable, for diagnostics only) and one 8-byte record per 64 KiB output
 *   block: the compressed offset of the block's first element and the masked CRC-32C of its decoded bytes. Block j's
 *   compressed bytes end where block j + 1's begin (n for the last); its decoded offset 65536 * j and length
 *   min(65536, dn - 65536 * j) are implied. sb_raw_table_bytes(nblocks) = 64 + 8 * nblocks. A table holds no pointers and
 *   may be copied or moved.
 *   A unit is seekable when Decoder::decompress returns Ok and every block decodes alone to the same bytes: a unit
 *   announcing more than 65,536 bytes that sb_decompress_batch_device_ws (same in_bytes, caps of at least dn) splits and
 *   decodes block-parallel with Ok (d_unit_blocks[i] > 0), or a unit announcing at most 65,536 bytes (0 included) that
 *   decodes Ok. Everything else (empty input, bad header, copies into an earlier block, elements across a block
 *   boundary, unblocked encoders, corrupt or truncated streams, and units over one block when the lengths sum past
 *   in_bytes) is not seekable.
 *   The tables are packed back to back in batch order into d_tables (device, 8-byte aligned, at least
 *   sb_raw_table_batch_bytes(count, in_bytes) bytes). d_table_offs (device, count + 1 entries) gets d_table_offs[0] = 0
 *   and d_table_offs[i + 1] = d_table_offs[i] + sb_raw_table_bytes(d_results[i].nchunks). d_results[i] is {Ok, dn,
 *   nblocks} for a seekable unit and {SB_E_INVALID{a=i, b=0, c=5}, 0, 0} otherwise; a unit that is not seekable gets a
 *   64-byte header only. Every table is byte-identical (padding included) to what a count == 1 build of that stream gives.
 * Scratch: sb_raw_table_build_batch_scratch_bytes(count, in_bytes), need not be zeroed. Stream ordered, no allocation, no
 * host synchronisation, and the same launches whatever count holds. Null pointers, count >= 2^31 and tables or scratch
 * that are too small are SB_E_INVALID with nothing launched; count == 0 does nothing. */
uint64_t sb_raw_table_bytes(uint32_t nblocks);
uint64_t sb_raw_table_batch_bytes(uint32_t count, uint64_t in_bytes);
uint64_t sb_raw_table_build_batch_scratch_bytes(uint32_t count, uint64_t in_bytes);
int sb_raw_table_build_batch_device_ws(const sb_batch* batch, uint64_t in_bytes, void* d_tables, uint64_t tables_bytes,
                                       uint64_t* d_table_offs, sb_frame_result* d_results, void* scratch,
                                       uint64_t scratch_bytes, void* stream, sb_error* err);
/* Byte ranges of many tabled raw streams in one call. The arguments mean what they mean for
 * sb_frame_table_decode_ranges_device_ws: stream u is d_ins[u][0 .. d_in_lens[u]) and d_tables[u] its raw seek table, and
 * range r asks for decoded bytes [d_lo[r], d_lo[r] + d_len[r]) of stream d_unit[r] into d_out_ptrs[r]. With
 * end = min(lo + len, dn), a range decodes exactly the blocks that overlap [lo, end) and checks each one's CRC against its
 * record. d_statuses[r] and d_out_lens[r], in priority order:
 *   1. d_unit[r] >= count: SB_E_INVALID{a=unit, b=count, c=1}, 0;
 *   2. d_tables[u] is not a raw table of this format, or was built over a stream of another length than d_in_lens[u]:
 *      SB_E_INVALID{a=d_in_lens[u], b=the table's n (0 if it is not a raw table), c=2}, 0;
 *   3. the stream is not seekable: SB_E_INVALID{a=u, b=0, c=5}, 0;
 *   4. a covered block fails, the first in stream order j, with out_len max(65536 * j, lo) - lo: SB_E_INVALID{a=j, b=0,
 *      c=3} when its record breaks the build's bounds (offsets non-decreasing, every block's bytes inside [hl, n), block
 *      count ceil(dn / 65536), dn < 2^32), SB_E_INVALID{a=j, b=0, c=4} when it does not decode to its CRC (the stream is
 *      not the one the table was built over);
 *   5. otherwise Ok; max(end - lo, 0) (a range past the end is a short read, like pread).
 *   For a seekable table built from stream S and read over S, every range is Ok and equals Decoder::decompress(S)[lo..end].
 *   No table content makes the call read outside a stream or write outside [out_r, out_r + max(end - lo, 0)), the
 *   staging or the scratch.
 * A block shared by several ranges is decoded once per range; the scratch, sb_raw_table_ranges_scratch_bytes(nranges)
 * bytes, holds 128 KiB of staging per range. Stream ordered, no allocation, no host synchronisation, and the same
 * launches whatever count and nranges; nranges == 0 does nothing. Null pointers that are needed, count or
 * nranges >= 2^31 and scratch that is too small are SB_E_INVALID with nothing launched. */
uint64_t sb_raw_table_ranges_scratch_bytes(uint32_t nranges);
int sb_raw_table_decode_ranges_device_ws(const void* const* d_tables, const uint8_t* const* d_ins,
                                         const uint64_t* d_in_lens, uint32_t count, const uint32_t* d_unit,
                                         const uint64_t* d_lo, const uint64_t* d_len, uint8_t* const* d_out_ptrs,
                                         uint64_t* d_out_lens, sb_error* d_statuses, uint32_t nranges, void* scratch,
                                         uint64_t scratch_bytes, void* stream, sb_error* err);

/* Gathers: many small ranges over tabled frame or raw streams in one call. The arguments are exactly those of
 * sb_frame_table_decode_ranges_device_ws / sb_raw_table_decode_ranges_device_ws, and so is the result: every range gets
 * the status, out_len and bytes [out_r, out_r + out_len) that call gives it, and nothing outside
 * [out_r, out_r + max(end - lo, 0)) is written. No table content makes the call read outside a stream or write outside
 * a range's buffer or the scratch. What differs is the cost:
 *   - an interior chunk or block (inside [lo, end) in full) decodes straight into its range's buffer, once per range
 *     that holds it, as in the range calls;
 *   - an edge chunk or block (the head or tail one, straddling lo or end) is decoded and CRC-checked once per call,
 *     however many ranges share it as an edge. A chunk that is an edge of more than 256 ranges is decoded once per group
 *     of at most 256 of them, so that one hot key does not serialise a call behind one warp;
 *   - a chunk that is interior to one range and an edge of another is decoded once in each role.
 * The scratch, sb_*_gather_scratch_bytes(nranges), is 108 bytes per range of bookkeeping (a hash table of the edges and
 * their per-chunk lists), a few KiB of scan tiles and alignment, and a staging pool of min(2 * nranges, 4096) slots of
 * 64 KiB, one per decoding warp: at most 128 * nranges + 256 MiB + 64 KiB bytes whatever nranges, and within 3 KiB of the
 * range calls' scratch for one range. Stream ordered, no allocation, no host synchronisation, and the same launches
 * whatever count, nranges and the sharing pattern; nranges == 0 does nothing. Null pointers that are needed,
 * count >= 2^31, nranges > 2^28 and scratch that is too small are SB_E_INVALID with nothing launched. */
uint64_t sb_frame_table_gather_scratch_bytes(uint32_t nranges);
int sb_frame_table_gather_device_ws(const void* const* d_tables, const uint8_t* const* d_ins, const uint64_t* d_in_lens,
                                    uint32_t count, const uint32_t* d_unit, const uint64_t* d_lo, const uint64_t* d_len,
                                    uint8_t* const* d_out_ptrs, uint64_t* d_out_lens, sb_error* d_statuses,
                                    uint32_t nranges, void* scratch, uint64_t scratch_bytes, void* stream, sb_error* err);
uint64_t sb_raw_table_gather_scratch_bytes(uint32_t nranges);
int sb_raw_table_gather_device_ws(const void* const* d_tables, const uint8_t* const* d_ins, const uint64_t* d_in_lens,
                                  uint32_t count, const uint32_t* d_unit, const uint64_t* d_lo, const uint64_t* d_len,
                                  uint8_t* const* d_out_ptrs, uint64_t* d_out_lens, sb_error* d_statuses,
                                  uint32_t nranges, void* scratch, uint64_t scratch_bytes, void* stream, sb_error* err);

/* Gathers over streams that stay in host memory. The arguments are exactly those of sb_frame_table_gather_device_ws /
 * sb_raw_table_gather_device_ws, and every range gets the status, out_len and bytes that call gives it over the same
 * tables and the same stream bytes. Nothing is written outside [out_r, out_r + max(end - lo, 0)) or the scratch, and the
 * call rules and SB_E_INVALID checks are the device gather's. The difference: d_ins[u] may be any address the device
 * reads at the same value, that is page-locked host memory mapped into the device's address space (cudaHostAlloc /
 * cudaMallocHost, torch pin_memory, cudaHostRegister) or device memory. sb_host_stream_check tells which addresses
 * qualify. Pageable host memory is undefined behaviour (a device fault) and must not be passed.
 * Cost: the warp that decodes a chunk or block first copies its compressed body from stream memory into a compressed
 * slot of its own, in 16-byte loads, and decodes from there. Each body the call decodes is read from stream memory once
 * per decode: an edge once per work item of at most 256 ranges, an interior chunk or block once per range holding it.
 * No other stream byte is read, with two exceptions that read in place: a raw block whose compressed bytes do not fit
 * a slot (only a wasteful encoder writes one; a legal block may spend 5 bytes per output byte), and the re-decode that
 * finds a failing chunk's status. The tables, outputs, ranges and scratch are device memory.
 * Scratch, exactly: sb_*_table_gather_scratch_bytes(nranges) + min(2 * nranges, 4096) * 76,544 bytes (one slot of
 * 76,490 bytes, the largest frame chunk body, rounded up to 256, per pool warp): at most
 * 128 * nranges + 4096 * (65,536 + 76,544) + 64 KiB bytes whatever the streams hold. */
uint64_t sb_frame_table_gather_host_streams_scratch_bytes(uint32_t nranges);
int sb_frame_table_gather_host_streams_ws(const void* const* d_tables, const uint8_t* const* d_ins,
                                          const uint64_t* d_in_lens, uint32_t count, const uint32_t* d_unit,
                                          const uint64_t* d_lo, const uint64_t* d_len, uint8_t* const* d_out_ptrs,
                                          uint64_t* d_out_lens, sb_error* d_statuses, uint32_t nranges, void* scratch,
                                          uint64_t scratch_bytes, void* stream, sb_error* err);
uint64_t sb_raw_table_gather_host_streams_scratch_bytes(uint32_t nranges);
int sb_raw_table_gather_host_streams_ws(const void* const* d_tables, const uint8_t* const* d_ins,
                                        const uint64_t* d_in_lens, uint32_t count, const uint32_t* d_unit,
                                        const uint64_t* d_lo, const uint64_t* d_len, uint8_t* const* d_out_ptrs,
                                        uint64_t* d_out_lens, sb_error* d_statuses, uint32_t nranges, void* scratch,
                                        uint64_t scratch_bytes, void* stream, sb_error* err);
/* Host only, no launch: Ok when p and p + n - 1 are both readable by the current device at the same address (page-locked
 * host memory mapped at that address, or device memory); n == 0 is Ok. Otherwise SB_E_INVALID{a = p, b = n, c = 6}. */
int sb_host_stream_check(const void* p, uint64_t n, sb_error* err);

/* Batch encoders that also write one seek table per unit, so what they write is seekable without a build. Each does
 * exactly what its untabled call does: output bytes, out_lens, statuses and (frame) d_chunk_offs are byte-identical to
 * sb_compress_batch_device_ws / sb_frame_encode_batch_device_ws with the same arguments, rejected units and the in_bytes
 * overflow (SB_E_INVALID{sum, in_bytes}) included. The tables are packed back to back in batch order into d_tables
 * (device, 8-byte aligned, at least sb_compress_tables_bytes / sb_frame_encode_tables_bytes(count, in_bytes) bytes);
 * d_table_offs (device, count + 1 entries) gets d_table_offs[0] = 0 and every table's end.
 *   Raw: unit i's table and d_results[i] are byte-identical, padding included, to what sb_raw_table_build_batch_device_ws
 *     (in_bytes at least the sum of out_lens) writes for out_i[0 .. out_lens[i]): {Ok, n, ceil(n / 65536)} and a seekable
 *     table for every written unit; a rejected unit (0 bytes) gets the not-seekable header with n = 0 and
 *     {SB_E_INVALID{a=i, b=0, c=5}, 0, 0}. One exception: a stream the build declines only because a K8 segment needs
 *     more than 1,024 merge elements (reason 3). There the encoder's table is still seekable and correct, since the
 *     encoder knows its own block starts.
 *   Frame: unit i's table and d_results[i] are byte-identical to what sb_frame_table_build_batch_device_ws (flags 0, a
 *     large enough max_chunks) writes for out_i[0 .. out_lens[i]). Empty and rejected units (0 bytes) get the table of
 *     an empty stream.
 * The records come from the encode itself: every block's compressed offset is a scan value of the encode, its decoded
 * offset is 65536 * j and its masked CRC-32C comes from the compress kernel's emitter warp. No output is read back.
 * Scratch: sb_compress_batch_tabled_scratch_bytes / sb_frame_encode_batch_tabled_scratch_bytes(count, in_bytes), need
 * not be zeroed. Stream ordered, no allocation, no host synchronisation, and the same launches whatever count holds (for
 * the frame call: one number with d_chunk_offs, one without). Null pointers (batch, out_lens, d_tables, d_table_offs,
 * d_results, scratch), count >= 2^31, a bound whose block count does not fit one launch and tables or scratch that are
 * too small are SB_E_INVALID with nothing launched; count == 0 does nothing. */
uint64_t sb_compress_tables_bytes(uint32_t count, uint64_t in_bytes);
uint64_t sb_compress_batch_tabled_scratch_bytes(uint32_t count, uint64_t in_bytes);
int sb_compress_batch_tabled_device_ws(const sb_batch* batch, uint64_t in_bytes, void* d_tables, uint64_t tables_bytes,
                                       uint64_t* d_table_offs, sb_frame_result* d_results, void* scratch,
                                       uint64_t scratch_bytes, void* stream, sb_error* err);
uint64_t sb_frame_encode_tables_bytes(uint32_t count, uint64_t in_bytes);
uint64_t sb_frame_encode_batch_tabled_scratch_bytes(uint32_t count, uint64_t in_bytes);
int sb_frame_encode_batch_tabled_device_ws(const sb_batch* batch, uint64_t in_bytes, uint64_t* d_chunk_offs,
                                           void* d_tables, uint64_t tables_bytes, uint64_t* d_table_offs,
                                           sb_frame_result* d_results, void* scratch, uint64_t scratch_bytes,
                                           void* stream, sb_error* err);

/* Chunk index of a frame stream in device memory, built in parallel on the device:
 * the offset of every chunk header in d_in[0..n) followed by n -- exactly the
 * d_chunk_offs that sb_frame_decode_device_ws accepts (max_chunks + 1 entries).
 * Only clean streams are indexed: the stream identifier (none when flags bit0,
 * a fragment), then data chunks only, covering the stream exactly. *d_count
 * (device) receives the number of chunks, or SB_FRAME_NOT_INDEXABLE for anything
 * else (skippable or padding chunks, a repeated identifier, reserved chunk types,
 * truncation, more than max_chunks chunks). Stream ordered, caller scratch of
 * sb_frame_index_scratch_bytes(n, max_chunks) bytes, no allocation. Index a
 * stream once to decode it many times, or to hand a rank a chunk range. */
#define SB_FRAME_NOT_INDEXABLE 0xFFFFFFFFu
uint64_t sb_frame_index_scratch_bytes(uint64_t n, uint32_t max_chunks);
int sb_frame_index_device_ws(const uint8_t* d_in, uint64_t n, uint32_t flags, uint64_t* d_chunk_offs, uint32_t max_chunks,
                             uint32_t* d_count, void* scratch, uint64_t scratch_bytes, void* stream, sb_error* err);

/* ---- resources -------------------------------------------------------------
 * The host entry points keep grow-only per-device pools (device staging, pinned
 * descriptors, streams, events): the first calls size them, the steady state
 * allocates nothing. sb_reserve sizes them ahead of time for waves of up to
 * wave_units units / wave_in_bytes input / wave_out_bytes output;
 * sb_alloc_count() = allocations + event/stream creations since load (a caller
 * can assert it stays flat). First use of a device is thread safe. */
int sb_reserve(size_t wave_units, size_t wave_in_bytes, size_t wave_out_bytes, sb_error* err);
uint64_t sb_alloc_count(void);
/* Pin the calling thread to the CPUs of the NUMA node of `device` (so that pinned staging it allocates afterwards
 * and its copies stay on the near socket). Returns the node, or -1 when the topology is not exposed. */
int sb_bind_host_thread_to_device_numa(int device);

/* ---- libsnappy-compatible C API ------------------------------------------
 * The four functions the reference's `snappy-cpp` crate binds
 * (snappy-cpp/src/lib.rs:66-88, snappy-c.h): linking the reference's test/ and
 * bench/ crates with `--features cpp` against this library runs their
 * cross-implementation tests on the GPU codec. 0 = SNAPPY_OK, 1 = INVALID_INPUT,
 * 2 = BUFFER_TOO_SMALL. */
int snappy_compress(const char* input, size_t input_length, char* compressed, size_t* compressed_length);
int snappy_uncompress(const char* compressed, size_t compressed_length, char* uncompressed, size_t* uncompressed_length);
size_t snappy_max_compressed_length(size_t source_length);
int snappy_uncompressed_length(const char* compressed, size_t compressed_length, size_t* result);

/* ---- misc ---------------------------------------------------------------- */
/* Number of kernel launches issued by this library since load (bench.py's
 * gpu_launches evidence). */
uint64_t sb_launch_count(void);
/* Device-side helper used by tests/bench: fills unit i (i < count) at
 * d_out + i*stride with text[off_i .. off_i+len), off_i = ((first+i)*mul) % (text_len-len). */
int sb_generate_blocks_device(const uint8_t* d_text, uint64_t text_len, uint8_t* d_out, uint64_t stride,
                              uint32_t len, uint64_t first, uint64_t count, uint64_t mul, void* stream, sb_error* err);
const char* sb_version(void);

#ifdef __cplusplus
}
#endif
#endif

"""Frame-format constants and one-shot helpers (reference src/frame.rs)."""
import ctypes as C

from . import _lib
from .error import from_c
from .raw import (HOST_BUILD_BYTES, _batch_encode, _check_ranges, _gather, _gathered, _host_streams, _ptr, _split,
                  _stored_tables, _validate_units, _windows)

MAX_BLOCK_SIZE = 1 << 16                      # src/lib.rs:97
MAX_COMPRESS_BLOCK_SIZE = 76490               # src/frame.rs:12
STREAM_IDENTIFIER = b"\xFF\x06\x00\x00sNaPpY"  # src/frame.rs:18
STREAM_BODY = b"sNaPpY"
CHUNK_HEADER_AND_CRC_SIZE = 8                 # src/frame.rs:26


def encode_chunks(data, include_ident: bool) -> bytes:
    """Chunks for `data` exactly as write::Inner::write emits them (src/write.rs:165-192)."""
    n = len(data)
    if n == 0:
        return STREAM_IDENTIFIER if include_ident else b""
    cap = _lib.lib().sb_frame_max_len(n)
    out = bytearray(cap)
    ip, k1 = _ptr(data)
    op, k2 = _ptr(out)
    m, e = C.c_size_t(0), _lib.SbError()
    if _lib.lib().sb_frame_encode_ex(ip, n, op, cap, C.byref(m), 1 if include_ident else 0, C.byref(e)):
        raise from_c(e)
    return bytes(out[:m.value])


def max_len(n: int) -> int:
    """sb_frame_max_len(n): the identifier and the largest chunk per started 64 KB slice."""
    return len(STREAM_IDENTIFIER) + (n + MAX_BLOCK_SIZE - 1) // MAX_BLOCK_SIZE * (CHUNK_HEADER_AND_CRC_SIZE +
                                                                                   MAX_COMPRESS_BLOCK_SIZE)


def encode_batch(units, tables=False) -> list:
    """Every unit as `FrameEncoder::new(vec![]).write_all(unit); into_inner()`, which is what sb_frame_encode returns: a
    complete framed stream per unit, b"" for an empty one. Units are bytes-like (bytes, bytearray, memoryview, numpy
    arrays). One sb_frame_encode_batch_device_ws call on the current torch stream encodes all of them; the inputs go to
    the device in one copy and the streams come back in one. Raises the first failing unit's error. tables=True makes
    the tabled call instead (sb_frame_encode_batch_tabled_device_ws) and returns (streams, tables): every stream's seek
    table as bytes, what TableReader would build for it, ready to be stored beside it and given to
    TableReader(..., tables=)."""
    return _batch_encode(units, lambda n: max_len(n) if max_len(n) <= 0xFFFFFFFF else 0, True, tables)


_FRAME_TABLE_MAGIC = 0x0001000042545342    # "BSTB", format version 1 (k13_frame_table.cuh)
MAX_BATCH_CHUNKS = (1 << 22) - 2             # the largest chunk table sb_frame_decode_batch_device_ws takes


def decode_batch(streams) -> list:
    """Every stream as `FrameDecoder::new(stream).read_to_end()`: one bytes object per stream, b"" for an empty one.
    Streams are bytes-like. The inputs go to the device in one copy and the decoded bytes come back in one; two
    sb_frame_decode_batch_device_ws calls on the current torch stream do the work: one with every cap 0, whose
    BufferTooSmall{0, need} sizes the outputs, then the decode. Raises the first failing stream's error."""
    import numpy as np
    import torch
    L = _lib.lib()
    views = [np.frombuffer(s, dtype=np.uint8) for s in streams]
    count = len(views)
    if count == 0:
        return []
    lens = [v.size for v in views]
    in_offs = np.zeros(count, dtype=np.int64)
    in_offs[1:] = np.cumsum(lens[:-1])
    host = np.empty(sum(lens) + 1, dtype=np.uint8)
    for o, v in zip(in_offs, views):
        host[o:o + v.size] = v
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.current_stream(dev).cuda_stream
    t_in = torch.from_numpy(host).to(dev)
    # out_lens (u32) and the statuses (sb_error, 32 bytes) of both calls, 8-byte aligned
    at_st = (4 * count + 7) // 8 * 8
    t_res = torch.empty(at_st + 32 * count, dtype=torch.uint8, device=dev)
    e = _lib.SbError()

    def call(out_offs, caps, out_base, max_chunks):
        desc = np.concatenate([in_offs + t_in.data_ptr(), out_offs + out_base,
                               np.array(lens + caps, dtype=np.uint32).view(np.int64)])
        t_desc = torch.from_numpy(desc).to(dev)
        b = _lib.SbBatch()
        b.in_ptrs, b.out_ptrs = t_desc.data_ptr(), t_desc.data_ptr() + 8 * count
        b.in_lens, b.out_caps = t_desc.data_ptr() + 16 * count, t_desc.data_ptr() + 20 * count
        b.out_lens, b.statuses, b.count = t_res.data_ptr(), t_res.data_ptr() + at_st, count
        need = L.sb_frame_decode_batch_scratch_bytes(count, sum(lens), max_chunks)
        t_scr = torch.empty(need, dtype=torch.uint8, device=dev)
        if L.sb_frame_decode_batch_device_ws(C.byref(b), sum(lens), 0, None, None, max_chunks, None, t_scr.data_ptr(),
                                             need, stream, C.byref(e)):
            raise from_c(e)
        return t_res.cpu().numpy()[at_st:].view(np.uint64).reshape(count, 4)

    zeros = np.zeros(count, dtype=np.int64)
    # the chunk table: a data chunk is at least 8 bytes, so n / 8 per stream always suffices
    max_chunks = min(sum(n // 1024 + 2 for n in lens), MAX_BATCH_CHUNKS)
    st = call(zeros, [0] * count, t_in.data_ptr(), max_chunks)
    if any(int(s[0]) & 0xFFFFFFFF == 202 and int(s[2]) == 1 for s in st):
        max_chunks = min(sum(n // 8 + 2 for n in lens), MAX_BATCH_CHUNKS)
        st = call(zeros, [0] * count, t_in.data_ptr(), max_chunks)
    caps = [int(s[2]) if int(s[0]) & 0xFFFFFFFF == 2 else 0 for s in st]   # BufferTooSmall{0, need}
    out_offs = np.zeros(count, dtype=np.int64)
    out_offs[1:] = np.cumsum(caps[:-1])
    t_out = torch.empty(sum(caps) + 1, dtype=torch.uint8, device=dev)
    st = call(out_offs, caps, t_out.data_ptr(), max_chunks)
    for s in st:
        if s[0] & 0xFFFFFFFF:
            raise from_c(_lib.SbError(int(s[0] & 0xFFFFFFFF), 0, int(s[1]), int(s[2]), int(s[3])))
    back = t_out.cpu().numpy()
    return [back[o:o + k].tobytes() for o, k in zip(out_offs, caps)]


def validate_batch(streams) -> list:
    """Every stream checked as `FrameDecoder::new(stream).read_to_end()` would check it, CRCs included, without its
    decoded bytes: one sb_frame_validate_batch_device_ws call on the current torch stream, with the chunk table sized
    and retried as decode_batch does. Streams are bytes-like; they go to the device in one copy and only out_lens and the
    statuses come back. Returns [(nbytes, error)]: the decoded length and None, or the bytes produced before the first
    error and that error (returned, not raised)."""
    import numpy as np
    import torch
    L = _lib.lib()
    lens = [memoryview(s).nbytes for s in streams]

    def run(b, in_bytes, t_res, stream):
        def call(max_chunks):
            need = L.sb_frame_validate_batch_scratch_bytes(b.count, in_bytes, max_chunks)
            t_scr = torch.empty(need, dtype=torch.uint8, device=t_res.device)
            e = _lib.SbError()
            if L.sb_frame_validate_batch_device_ws(C.byref(b), in_bytes, 0, None, None, max_chunks, None, t_scr.data_ptr(),
                                                   need, stream, C.byref(e)):
                raise from_c(e)
            return t_res.cpu().numpy()

        at_st = (4 * b.count + 7) // 8 * 8
        back = call(min(sum(n // 1024 + 2 for n in lens), MAX_BATCH_CHUNKS))
        if any(int(s[0]) & 0xFFFFFFFF == 202 and int(s[2]) == 1 for s in back[at_st:].view(np.uint64).reshape(-1, 4)):
            back = call(min(sum(n // 8 + 2 for n in lens), MAX_BATCH_CHUNKS))
        return back

    return _validate_units(streams, run)


def decode_all(stream) -> bytes:
    """read::FrameDecoder::new(stream).read_to_end() (src/read.rs:104-239)."""
    n = len(stream)
    ip, k1 = _ptr(stream) if n else (None, None)
    m, e = C.c_size_t(0), _lib.SbError()
    L = _lib.lib()
    if L.sb_frame_decode(ip, n, None, 0, C.byref(m), C.byref(e)):
        raise from_c(e)
    out = bytearray(max(m.value, 1))
    op, k2 = _ptr(out)
    if L.sb_frame_decode(ip, n, op, m.value, C.byref(m), C.byref(e)):
        raise from_c(e)
    return bytes(out[:m.value])


def decode_all_partial(stream):
    """Like decode_all, but a failing stream yields (bytes produced before the failure, the exception) instead of
    raising: what a reader delivers before its n-th read fails."""
    n = len(stream)
    ip, k1 = _ptr(stream) if n else (None, None)
    m, e = C.c_size_t(0), _lib.SbError()
    L = _lib.lib()
    if L.sb_frame_decode(ip, n, None, 0, C.byref(m), C.byref(e)):
        return b"", from_c(e)
    out = bytearray(max(m.value, 1))
    op, k2 = _ptr(out)
    rc = L.sb_frame_decode(ip, n, op, m.value, C.byref(m), C.byref(e))
    return bytes(out[:m.value]), (from_c(e) if rc else None)


class RangeReader:
    """Random access to the decoded bytes of one frame stream on the device: `read(lo, n)` returns decoded bytes
    [lo, lo + n) as `FrameDecoder::new(stream).read_to_end()` would, after decoding and checksumming only the chunks
    those bytes come from. A range past the end is a short read, like `pread`. The stream is a bytes-like object
    (uploaded once) or a CUDA uint8 tensor (used as it is, and kept alive). It is indexed once on the device; a stream the
    indexer declines (padding or skippable chunks, a repeated identifier, ...) is walked by one thread on every call.
    fragment: the stream has no identifier. Calls run on the current torch stream and wait for their results."""

    RANGES_PER_CALL = 4096                    # 128 KiB of staging per range: 512 MiB per call at most
    BYTES_PER_CALL = 1 << 30                  # output bytes one call gathers (a single larger range gets its own call)

    def __init__(self, stream, fragment=False):
        import numpy as np
        import torch
        L = _lib.lib()
        self._dev = torch.device("cuda", torch.cuda.current_device())
        if isinstance(stream, torch.Tensor):
            if not stream.is_cuda or stream.dtype != torch.uint8 or stream.dim() != 1 or not stream.is_contiguous():
                raise ValueError("RangeReader takes a contiguous 1-D CUDA uint8 tensor")
            self._in = stream
        else:
            self._in = torch.from_numpy(np.frombuffer(stream, dtype=np.uint8).copy()).to(self._dev)
        self._n, self._flags = self._in.numel(), 1 if fragment else 0
        self._cuda = torch.cuda.current_stream(self._dev).cuda_stream
        # the chunk table: encoder chunks hold 64 KiB each, and a data chunk is at least 8 bytes whatever wrote it
        self._max_chunks = min(self._n // 1024 + 16, MAX_BATCH_CHUNKS)
        self._index()
        res = self._call([])[2]
        if res.status.code == 202 and res.status.b == 1:
            self._max_chunks = min(self._n // 8 + 16, MAX_BATCH_CHUNKS)
            self._index()
            res = self._call([])[2]
        self._result = res
        self.total = int(res.bytes)

    def _index(self):
        import numpy as np
        import torch
        L = _lib.lib()
        self._offs = torch.empty(self._max_chunks + 1, dtype=torch.int64, device=self._dev)
        count = torch.empty(1, dtype=torch.int32, device=self._dev)
        need = L.sb_frame_index_scratch_bytes(self._n, self._max_chunks)
        scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
        e = _lib.SbError()
        if L.sb_frame_index_device_ws(self._in.data_ptr(), self._n, self._flags, self._offs.data_ptr(), self._max_chunks,
                                      count.data_ptr(), scr.data_ptr(), need, self._cuda, C.byref(e)):
            raise from_c(e)
        c = int(count.cpu().numpy().view(np.uint32)[0])
        self._nchunks = None if c == 0xFFFFFFFF else c        # SB_FRAME_NOT_INDEXABLE: walked

    def _call(self, ranges):
        """One sb_frame_decode_ranges_device_ws call: (out_lens, statuses, stream result, output tensor, offsets)."""
        import numpy as np
        import torch
        L = _lib.lib()
        k = len(ranges)
        # a buffer needs only what the stream can give the range: nothing is written past min(lo + n, total)
        total = getattr(self, "total", 0)
        room = [max(0, min(n, total - lo)) for lo, n in ranges]
        offs = np.zeros(k, dtype=np.int64)
        if k:
            offs[1:] = np.cumsum(room[:-1])
        t_out = torch.empty(sum(room) + 1, dtype=torch.uint8, device=self._dev)
        desc = np.array([lo for lo, _ in ranges] + [n for _, n in ranges], dtype=np.uint64).view(np.int64)
        t_desc = torch.from_numpy(np.concatenate([desc, offs + t_out.data_ptr()])).to(self._dev)
        t_res = torch.zeros(5 * k + 6, dtype=torch.int64, device=self._dev)   # out_lens, statuses, the stream result
        need = L.sb_frame_decode_ranges_scratch_bytes(self._max_chunks, k)
        scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
        e = _lib.SbError()
        p = t_desc.data_ptr()
        if L.sb_frame_decode_ranges_device_ws(self._in.data_ptr(), self._n,
                                              self._offs.data_ptr() if self._nchunks is not None else None,
                                              self._nchunks or 0, self._flags, p, p + 8 * k, p + 16 * k, t_res.data_ptr(),
                                              t_res.data_ptr() + 8 * k, k, t_res.data_ptr() + 40 * k, scr.data_ptr(), need,
                                              self._max_chunks, self._cuda, C.byref(e)):
            raise from_c(e)
        back = t_res.cpu().numpy().view(np.uint64)
        res = _lib.SbFrameResult.from_buffer_copy(back[5 * k:].tobytes()[:C.sizeof(_lib.SbFrameResult)])
        return back[:k], back[k:5 * k].reshape(k, 4), res, t_out, offs

    def __len__(self):
        return self.total

    def read(self, lo: int, n: int) -> bytes:
        """Decoded bytes [lo, lo + n), fewer at the end of the stream."""
        return self.read_ranges([(lo, n)])[0]

    def read_ranges(self, ranges) -> list:
        """One bytes object per (lo, n) range. Ranges may be empty, unsorted, overlapping or repeated; each call to the
        library takes a group of them whose staging and output stay bounded. Raises the first failing range's error."""
        ranges = [(int(lo), int(n)) for lo, n in ranges]
        for lo, n in ranges:
            if lo < 0 or n < 0 or lo + n > 0xFFFFFFFFFFFFFFFF:
                raise ValueError("range (%d, %d) is not within 64-bit offsets" % (lo, n))
        out, i = [], 0
        while i < len(ranges):
            j, size = i, 0
            while j < len(ranges) and j - i < self.RANGES_PER_CALL:
                room = max(0, min(ranges[j][1], self.total - ranges[j][0]))
                if j > i and size + room > self.BYTES_PER_CALL:
                    break
                size += room
                j += 1
            lens, sts, _, t_out, offs = self._call(ranges[i:j])
            for s in sts:
                if s[0] & 0xFFFFFFFF:
                    raise from_c(_lib.SbError(int(s[0] & 0xFFFFFFFF), 0, int(s[1]), int(s[2]), int(s[3])))
            back = t_out.cpu().numpy()
            out += [back[o:o + int(m)].tobytes() for o, m in zip(offs, lens)]
            i = j
        return out


class TableReader:
    """Random access to the decoded bytes of many frame streams on the device. Each stream gets a seek table, built once
    on the device: a pointer-free list of its data chunks with their decoded offsets. The tables are built in batch
    calls (sb_frame_table_build_batch_device_ws), one per group of streams whatever their number. `read_ranges([(i, lo, n), ...])`
    then serves ranges of any of the streams in one library call per group, decoding and checksumming only the chunks
    they cover, with no pass over any stream's headers. Every range gives what `RangeReader(streams[i]).read(lo, n)`
    gives. A stream is a bytes-like object (uploaded once) or a contiguous 1-D CUDA uint8 tensor (kept alive).
    fragment: the streams have no identifier. Calls run on the current torch stream and wait for their results.
    tables: the streams' stored seek tables (from encode_batch(..., tables=True) or an earlier build), bytes-like or
    CUDA uint8 tensors, instead of a build. They are uploaded in one copy and no build runs; a table whose header does
    not match its stream's length raises ValueError. A table of another stream of the same length gives the reads over
    it a chunk's checksum error, never wrong bytes.
    host: the streams stay in pinned host memory (bytes-like ones copied once into one pinned buffer, pinned CPU uint8
    tensors kept alive; unpinned CPU and CUDA tensors raise ValueError), so a corpus larger than the device can be read.
    Only the tables live on the device: they are built from uploads of at most HOST_BUILD_BYTES of streams at a time.
    Reads go through sb_frame_table_gather_host_streams_ws, which copies over PCIe only the compressed chunks it
    decodes; read_ranges is then the gather, split. Results and errors are those of a reader without host."""

    RANGES_PER_CALL = RangeReader.RANGES_PER_CALL
    BYTES_PER_CALL = RangeReader.BYTES_PER_CALL

    def __init__(self, streams, fragment=False, tables=None, host=False):
        import numpy as np
        import torch
        self._dev = torch.device("cuda", torch.cuda.current_device())
        self._cuda = torch.cuda.current_stream(self._dev).cuda_stream
        self._host = bool(host)
        self._ins, host = ([], []) if not self._host else (_host_streams(streams), [])
        for s in streams if not self._host else ():
            if isinstance(s, torch.Tensor):
                if not s.is_cuda or s.dtype != torch.uint8 or s.dim() != 1 or not s.is_contiguous():
                    raise ValueError("TableReader takes contiguous 1-D CUDA uint8 tensors")
                self._ins.append(s)
            else:
                host.append((len(self._ins), np.frombuffer(s, dtype=np.uint8)))
                self._ins.append(None)
        if host:                                                         # the bytes-like streams go up in one copy
            at = np.cumsum([0] + [v.size for _, v in host])
            cat = np.empty(int(at[-1]) + 1, dtype=np.uint8)
            for (_, v), o in zip(host, at):
                cat[o:o + v.size] = v
            t_all = torch.from_numpy(cat).to(self._dev)
            for (i, v), o in zip(host, at):
                self._ins[i] = t_all[int(o):int(o) + v.size]
        flags = 1 if fragment else 0
        count = len(self._ins)
        lens = [t.numel() for t in self._ins]
        self._bufs = []                                                  # the tables live in these
        if tables is not None:
            self._bufs, heads = _stored_tables(tables, lens, self._dev, _FRAME_TABLE_MAGIC, 32,
                                               lambda w: int(w[3]) & 0xFFFFFFFF)
            self.lengths = [int(w[2]) for w in heads]
            self._keep_tables([t.data_ptr() for t in self._bufs], lens)
            return
        ptrs, results = [0] * count, [None] * count
        groups = _windows(range(count), lens, HOST_BUILD_BYTES) if self._host else [list(range(count))]
        for g in groups:                                                 # host streams: one uploaded window at a time
            ins = {i: self._ins[i].to(self._dev) for i in g} if self._host else self._ins
            # a stream that fits an sb_batch unit is tabled in a batch call; a longer one gets a build of its own
            for i, t, r in zip(*self._build([i for i in g if lens[i] > 0xFFFFFFFF], flags, ins)):
                self._bufs.append(t)
                ptrs[i], results[i] = t.data_ptr(), r
            # the chunk table as RangeReader sizes it: encoder chunks hold 64 KiB, and any data chunk is at least 8
            # bytes. Streams that did not fit the first time are built again with the larger bound.
            todo = [i for i in g if lens[i] <= 0xFFFFFFFF]
            for per in (1024, 8):
                for i, p, r in self._build_batch(todo, [min(lens[i] // per + 16, MAX_BATCH_CHUNKS) for i in todo], flags,
                                                 ins):
                    ptrs[i], results[i] = p, r
                todo = [i for i in todo if results[i].status.code == 202 and results[i].status.b == 1]
            del ins
        self.lengths = [int(r.bytes) for r in results]
        self._keep_tables(ptrs, lens)

    def _keep_tables(self, ptrs, lens):
        """The device arrays of table addresses, stream addresses and stream lengths every read passes."""
        import numpy as np
        import torch
        to64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).to(self._dev)
        self._t_tables = to64(ptrs + [0])
        self._t_ins = to64([t.data_ptr() for t in self._ins] + [0])
        self._t_lens = to64(lens + [0])

    def _build_batch(self, which, caps, flags, streams):
        """sb_frame_table_build_batch_device_ws over groups of `streams` (device tensors by stream index) whose chunk
        tables (caps) sum to at most MAX_BATCH_CHUNKS: one call and one wait per group, whatever the number of streams.
        A group's tables stay in one buffer cut to their packed size. Yields (stream, its table's address, its result)
        for every stream."""
        import numpy as np
        import torch
        L = _lib.lib()
        groups, cur, total = [], [], 0
        for i, c in zip(which, caps):
            if cur and total + c > MAX_BATCH_CHUNKS:
                groups.append((cur, total))
                cur, total = [], 0
            cur.append(i)
            total += c
        if cur:
            groups.append((cur, total))
        rsz = C.sizeof(_lib.SbFrameResult)
        for g, max_chunks in groups:
            k = len(g)
            ins = [streams[i] for i in g]
            in_bytes = sum(t.numel() for t in ins)
            desc = np.concatenate([np.array([t.data_ptr() for t in ins], dtype=np.uint64).view(np.int64),
                                   np.array([t.numel() for t in ins] + [0] * (k % 2), dtype=np.uint32).view(np.int64)])
            t_desc = torch.from_numpy(desc).to(self._dev)
            b = _lib.SbBatch()
            b.in_ptrs, b.in_lens, b.count = t_desc.data_ptr(), t_desc.data_ptr() + 8 * k, k
            tb = L.sb_frame_table_batch_bytes(k, max_chunks)
            t_tab = torch.empty(tb, dtype=torch.uint8, device=self._dev)
            t_res = torch.empty(8 * (k + 1) + rsz * k, dtype=torch.uint8, device=self._dev)   # offsets, then results
            need = L.sb_frame_table_build_batch_scratch_bytes(k, in_bytes, max_chunks)
            scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
            e = _lib.SbError()
            if L.sb_frame_table_build_batch_device_ws(C.byref(b), in_bytes, flags, None, None, max_chunks,
                                                      t_tab.data_ptr(), tb, t_res.data_ptr(),
                                                      t_res.data_ptr() + 8 * (k + 1), scr.data_ptr(), need, self._cuda,
                                                      C.byref(e)):
                raise from_c(e)
            back = t_res.cpu().numpy()
            offs = back[:8 * (k + 1)].view(np.uint64)
            kept = t_tab[:int(offs[k])].clone()
            self._bufs.append(kept)
            raw = back[8 * (k + 1):].tobytes()
            for j, i in enumerate(g):
                yield i, kept.data_ptr() + int(offs[j]), _lib.SbFrameResult.from_buffer_copy(raw[j * rsz:(j + 1) * rsz])

    def _build(self, which, flags, streams):
        """A table per stream by sb_frame_table_build_device_ws (streams too long for a batch unit), its chunk table
        sized as RangeReader sizes it and built once more when too small: (streams, tables cut to size, results)."""
        L = _lib.lib()
        if not which:
            return [], [], []
        caps = [min(streams[i].numel() // 1024 + 16, MAX_BATCH_CHUNKS) for i in which]
        tables, results = self._build_each(which, caps, flags, streams)
        for j, i in enumerate(which):
            if results[j].status.code == 202 and results[j].status.b == 1:
                more, res2 = self._build_each([i], [min(streams[i].numel() // 8 + 16, MAX_BATCH_CHUNKS)], flags,
                                              streams)
                tables[j], results[j] = more[0], res2[0]
        return which, [t[:L.sb_frame_table_bytes(r.nchunks)].clone() for t, r in zip(tables, results)], results

    def _build_each(self, which, caps, flags, streams):
        """One sb_frame_table_build_device_ws per stream, one wait for all: (tables, results)."""
        import numpy as np
        import torch
        L = _lib.lib()
        which = list(which)
        need = max([L.sb_frame_table_build_scratch_bytes(c) for c in caps] + [1])
        scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
        rsz = C.sizeof(_lib.SbFrameResult)
        t_res = torch.zeros(max(len(which), 1) * rsz, dtype=torch.uint8, device=self._dev)
        tables = []
        for j, (i, cap) in enumerate(zip(which, caps)):
            t_in = streams[i]
            tb = L.sb_frame_table_bytes(cap)
            table = torch.empty(tb, dtype=torch.uint8, device=self._dev)
            e = _lib.SbError()
            if L.sb_frame_table_build_device_ws(t_in.data_ptr(), t_in.numel(), None, 0, flags, table.data_ptr(), tb, cap,
                                                t_res.data_ptr() + j * rsz, scr.data_ptr(), need, self._cuda, C.byref(e)):
                raise from_c(e)
            tables.append(table)
        back = t_res.cpu().numpy().tobytes()
        return tables, [_lib.SbFrameResult.from_buffer_copy(back[j * rsz:(j + 1) * rsz]) for j in range(len(which))]

    def __len__(self):
        return len(self._ins)

    def _call(self, ranges):
        """One sb_frame_table_decode_ranges_device_ws call: (out_lens, statuses, output tensor, offsets)."""
        import numpy as np
        import torch
        L = _lib.lib()
        k = len(ranges)
        room = [max(0, min(n, self.lengths[i] - lo)) for i, lo, n in ranges]
        offs = np.zeros(k, dtype=np.int64)
        if k:
            offs[1:] = np.cumsum(room[:-1])
        t_out = torch.empty(sum(room) + 1, dtype=torch.uint8, device=self._dev)
        desc = np.array([lo for _, lo, _ in ranges] + [n for _, _, n in ranges], dtype=np.uint64).view(np.int64)
        units = np.array([i for i, _, _ in ranges] + [0], dtype=np.uint32).view(np.int32)
        t_desc = torch.from_numpy(np.concatenate([desc, offs + t_out.data_ptr()])).to(self._dev)
        t_unit = torch.from_numpy(units).to(self._dev)
        t_res = torch.zeros(5 * k, dtype=torch.int64, device=self._dev)       # out_lens, statuses
        need = L.sb_frame_table_ranges_scratch_bytes(k)
        scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
        e = _lib.SbError()
        p = t_desc.data_ptr()
        if L.sb_frame_table_decode_ranges_device_ws(self._t_tables.data_ptr(), self._t_ins.data_ptr(),
                                                    self._t_lens.data_ptr(), len(self._ins), t_unit.data_ptr(), p,
                                                    p + 8 * k, p + 16 * k, t_res.data_ptr(), t_res.data_ptr() + 8 * k, k,
                                                    scr.data_ptr(), need, self._cuda, C.byref(e)):
            raise from_c(e)
        back = t_res.cpu().numpy().view(np.uint64)
        return back[:k], back[k:5 * k].reshape(k, 4), t_out, offs

    def read(self, i: int, lo: int, n: int) -> bytes:
        """Decoded bytes [lo, lo + n) of stream i, fewer at the end of the stream."""
        return self.read_ranges([(i, lo, n)])[0]

    def read_ranges(self, ranges) -> list:
        """One bytes object per (i, lo, n) range of stream i. Ranges may mix streams in any order and be empty,
        unsorted, overlapping or repeated; each library call takes a group of them whose staging and output stay
        bounded. Raises the first failing range's error. With host streams this is the gather, split."""
        if self._host:
            return _split(*self.gather(ranges))
        ranges = [(int(i), int(lo), int(n)) for i, lo, n in ranges]
        for i, lo, n in ranges:
            if not 0 <= i < len(self._ins):
                raise IndexError("stream %d of %d" % (i, len(self._ins)))
            if lo < 0 or n < 0 or lo + n > 0xFFFFFFFFFFFFFFFF:
                raise ValueError("range (%d, %d) is not within 64-bit offsets" % (lo, n))
        out, a = [], 0
        while a < len(ranges):
            b, size = a, 0
            while b < len(ranges) and b - a < self.RANGES_PER_CALL:
                i, lo, n = ranges[b]
                room = max(0, min(n, self.lengths[i] - lo))
                if b > a and size + room > self.BYTES_PER_CALL:
                    break
                size += room
                b += 1
            lens, sts, t_out, offs = self._call(ranges[a:b])
            for s in sts:
                if s[0] & 0xFFFFFFFF:
                    raise from_c(_lib.SbError(int(s[0] & 0xFFFFFFFF), 0, int(s[1]), int(s[2]), int(s[3])))
            back = t_out.cpu().numpy()
            out += [back[o:o + int(m)].tobytes() for o, m in zip(offs, lens)]
            a = b
        return out

    def gather(self, ranges):
        """Every (i, lo, n) range of stream i gathered on the device: (data, offsets), data one CUDA uint8 tensor with
        the ranges back to back and offsets an int64 array of len(ranges) + 1 entries, data[offsets[j]:offsets[j + 1]]
        being read_ranges(ranges)[j]. Ranges may be as read_ranges takes them. The calls
        (sb_frame_table_gather_device_ws) decode a chunk shared by many ranges as an edge once per call, and take up to
        GATHER_RANGES_PER_CALL ranges and BYTES_PER_CALL output bytes each. Raises the first failing range's error, as
        read_ranges does."""
        import torch
        ranges = _check_ranges(ranges, len(self._ins))
        rooms = [max(0, min(n, self.lengths[i] - lo)) for i, lo, n in ranges]
        offs = _gathered(rooms)
        data = torch.empty(int(offs[-1]), dtype=torch.uint8, device=self._dev)
        bad = _gather(self, "frame", ranges, rooms, data, offs[:-1]) if ranges else None
        if bad:
            raise bad[1]
        return data, offs

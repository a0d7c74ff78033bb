"""`snap::raw` mirrored over the C ABI (reference src/raw.rs:13-14).

`Encoder.compress/compress_vec`, `Decoder.decompress/decompress_vec`,
`max_compress_len`, `decompress_len` keep the reference's argument meaning and
error behaviour (src/compress.rs:42-169, src/decompress.rs:30-110); the work is
done by the CUDA kernels behind `sb_compress` / `sb_decompress`.
"""
import ctypes as C

from . import _lib
from .error import from_c


def _ptr(buf):
    """address of a bytes-like object without copying (bytes, bytearray, memoryview, numpy)."""
    if isinstance(buf, bytes):
        return C.cast(C.c_char_p(buf), C.c_void_p).value, buf
    mv = memoryview(buf)
    if mv.readonly:
        b = bytes(mv)
        return C.cast(C.c_char_p(b), C.c_void_p).value, b
    arr = (C.c_char * mv.nbytes).from_buffer(mv)
    return C.addressof(arr), arr


def max_compress_len(input_len: int) -> int:
    return _lib.lib().sb_max_compress_len(input_len)


def decompress_len(data) -> int:
    p, keep = _ptr(data)
    n, e = C.c_size_t(0), _lib.SbError()
    if _lib.lib().sb_decompress_len(p, len(data), C.byref(n), C.byref(e)):
        raise from_c(e)
    return n.value


class Encoder:
    """snap::raw::Encoder (src/compress.rs:67-170)."""

    def compress(self, input, output) -> int:
        ip, k1 = _ptr(input)
        op, k2 = _ptr(output)
        n, e = C.c_size_t(0), _lib.SbError()
        if _lib.lib().sb_compress(ip, len(input), op, len(output), C.byref(n), C.byref(e)):
            raise from_c(e)
        return n.value

    def compress_vec(self, input) -> bytes:
        buf = bytearray(max(max_compress_len(len(input)), 1))
        n = self.compress(input, buf)
        return bytes(buf[:n])


class Decoder:
    """snap::raw::Decoder (src/decompress.rs:45-111)."""

    def decompress(self, input, output) -> int:
        ip, k1 = _ptr(input)
        op, k2 = _ptr(output) if len(output) else (None, None)
        n, e = C.c_size_t(0), _lib.SbError()
        if _lib.lib().sb_decompress(ip, len(input), op, len(output), C.byref(n), C.byref(e)):
            raise from_c(e)
        return n.value

    def decompress_vec(self, input) -> bytes:
        buf = bytearray(decompress_len(input))
        n = self.decompress(input, buf)
        return bytes(buf[:n])


def validate(data) -> int:
    """The decoded length of a raw stream, found without decoding it into memory (sb_validate); raises exactly what
    `Decoder().decompress_vec(data)` raises."""
    p, keep = _ptr(data) if len(data) else (None, None)
    n, e = C.c_size_t(0), _lib.SbError()
    if _lib.lib().sb_validate(p, len(data), C.byref(n), C.byref(e)):
        raise from_c(e)
    return n.value


def crc32c_masked(data) -> int:
    """crc32::CheckSummer::crc32c_masked (src/crc32.rs:35-38), computed on the GPU."""
    p, keep = _ptr(data) if len(data) else (None, None)
    out, e = C.c_uint32(0), _lib.SbError()
    if _lib.lib().sb_crc32c_masked(p, len(data), C.byref(out), C.byref(e)):
        raise from_c(e)
    return out.value


_RAW_TABLE_MAGIC = 0x0001000042545352      # "RSTB", format version 1 (k15_raw_table.cuh)


def _batch_encode(units, cap_of, frame, tables):
    """One sb_compress_batch_device_ws (frame: sb_frame_encode_batch_device_ws) call over bytes-like units, or its tabled
    form: the inputs go to the device in one copy, the streams (and tables) come back in one. cap_of(n) is the unit's
    cap, 0 for a unit the call rejects without writing. Raises the first failing unit's error."""
    import numpy as np
    import torch
    L = _lib.lib()
    views = [np.frombuffer(u, dtype=np.uint8) for u in units]
    count = len(views)
    if count == 0:
        return ([], []) if tables else []
    lens = [v.size for v in views]
    caps = [cap_of(n) for n in lens]
    in_offs = np.zeros(count, dtype=np.int64)
    in_offs[1:] = np.cumsum(lens[:-1])
    host = np.empty(sum(lens) + 1, dtype=np.uint8)
    for o, v in zip(in_offs, views):
        host[o:o + v.size] = v
    out_offs = np.zeros(count, dtype=np.int64)
    out_offs[1:] = np.cumsum(caps[:-1])
    # one device buffer holds the streams, then out_lens (u32) and the statuses (sb_error, 32 bytes), 8-byte aligned
    at_lens = (sum(caps) + 7) // 8 * 8
    at_st = at_lens + (4 * count + 7) // 8 * 8
    dev = torch.device("cuda", torch.cuda.current_device())
    t_in = torch.from_numpy(host).to(dev)
    t_out = torch.empty(at_st + 32 * count, dtype=torch.uint8, device=dev)
    desc = np.concatenate([in_offs + t_in.data_ptr(), out_offs + t_out.data_ptr(),
                           np.array(lens + [c if c else 0xFFFFFFFF * frame for c in caps], dtype=np.uint32).view(np.int64)])
    t_desc = torch.from_numpy(desc).to(dev)
    b = _lib.SbBatch()
    b.in_ptrs, b.out_ptrs = t_desc.data_ptr(), t_desc.data_ptr() + 8 * count
    b.in_lens, b.out_caps = t_desc.data_ptr() + 16 * count, t_desc.data_ptr() + 20 * count
    b.out_lens, b.statuses, b.count = t_out.data_ptr() + at_lens, t_out.data_ptr() + at_st, count
    in_bytes = sum(n for n, c in zip(lens, caps) if n > 65536 and c)
    stream = torch.cuda.current_stream(dev).cuda_stream
    e = _lib.SbError()
    if tables:
        tb = (L.sb_frame_encode_tables_bytes if frame else L.sb_compress_tables_bytes)(count, in_bytes)
        need = (L.sb_frame_encode_batch_tabled_scratch_bytes if frame else L.sb_compress_batch_tabled_scratch_bytes)(
            count, in_bytes)
        t_scr = torch.empty(need, dtype=torch.uint8, device=dev)
        t_tab = torch.empty(tb + 8 * (count + 1) + C.sizeof(_lib.SbFrameResult) * count, dtype=torch.uint8, device=dev)
        p = t_tab.data_ptr()
        args = (p, tb, p + tb, p + tb + 8 * (count + 1), t_scr.data_ptr(), need, stream, C.byref(e))
        rc = L.sb_frame_encode_batch_tabled_device_ws(C.byref(b), in_bytes, None, *args) if frame else \
            L.sb_compress_batch_tabled_device_ws(C.byref(b), in_bytes, *args)
    else:
        need = (L.sb_frame_encode_batch_scratch_bytes if frame else L.sb_compress_batch_scratch_bytes)(count, in_bytes)
        t_scr = torch.empty(need, dtype=torch.uint8, device=dev)
        rc = L.sb_frame_encode_batch_device_ws(C.byref(b), in_bytes, None, t_scr.data_ptr(), need, stream, C.byref(e)) \
            if frame else L.sb_compress_batch_device_ws(C.byref(b), in_bytes, t_scr.data_ptr(), need, stream, C.byref(e))
    if rc:
        raise from_c(e)
    back = t_out.cpu().numpy()
    out_lens = back[at_lens:at_lens + 4 * count].view(np.uint32)
    for st in back[at_st:].view(np.uint64).reshape(count, 4):
        if st[0] & 0xFFFFFFFF:
            raise from_c(_lib.SbError(int(st[0] & 0xFFFFFFFF), 0, int(st[1]), int(st[2]), int(st[3])))
    streams = [back[o:o + k].tobytes() for o, k in zip(out_offs, out_lens)]
    if not tables:
        return streams
    offs = t_tab[tb:tb + 8 * (count + 1)].cpu().numpy().view(np.uint64)
    packed = t_tab[:int(offs[count])].cpu().numpy()
    return streams, [packed[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(count)]


def compress_batch(units, tables=False):
    """Every unit as `Encoder().compress_vec(unit)` returns it, in one sb_compress_batch_device_ws call on the current
    torch stream. Units are bytes-like (bytes, bytearray, memoryview, numpy arrays); the inputs go to the device in one
    copy and the streams come back in one. Raises the first failing unit's error. tables=True makes the tabled call
    instead (sb_compress_batch_tabled_device_ws) and returns (streams, tables): every stream's raw seek table as
    bytes, what TableReader would build for it, ready to be stored beside it and given to TableReader(..., tables=)."""
    return _batch_encode(units, lambda n: max_compress_len(n) if n < 0xFFFFFFFF else 0, False, tables)


def _validate_units(units, run):
    """Uploads bytes-like units with their descriptors in one copy, makes the validation call run(batch, in_bytes,
    results, stream) on the current torch stream (it returns the results' device tensor to read, or raises), and
    returns [(nbytes, error or None)] from one download of out_lens and the statuses."""
    import numpy as np
    import torch
    views = [np.frombuffer(u, dtype=np.uint8) for u in units]
    count = len(views)
    if count == 0:
        return []
    lens = [v.size for v in views]
    in_offs = np.zeros(count, dtype=np.int64)
    in_offs[1:] = np.cumsum(lens[:-1])
    at_desc = (sum(lens) + 7) // 8 * 8                       # in_ptrs (u64), then in_lens (u32)
    dev = torch.device("cuda", torch.cuda.current_device())
    t_in = torch.empty(at_desc + 12 * count, dtype=torch.uint8, device=dev)
    host = np.zeros(at_desc + 12 * count, dtype=np.uint8)
    for o, v in zip(in_offs, views):
        host[o:o + v.size] = v
    host[at_desc:at_desc + 8 * count] = (in_offs + t_in.data_ptr()).view(np.uint8)
    host[at_desc + 8 * count:] = np.array(lens, dtype=np.uint32).view(np.uint8)
    t_in.copy_(torch.from_numpy(host))
    # out_lens (u32) and the statuses (sb_error, 32 bytes), 8-byte aligned
    at_st = (4 * count + 7) // 8 * 8
    t_res = torch.empty(at_st + 32 * count, dtype=torch.uint8, device=dev)
    b = _lib.SbBatch()
    b.in_ptrs, b.in_lens = t_in.data_ptr() + at_desc, t_in.data_ptr() + at_desc + 8 * count
    b.out_lens, b.statuses, b.count = t_res.data_ptr(), t_res.data_ptr() + at_st, count
    back = run(b, sum(lens), t_res, torch.cuda.current_stream(dev).cuda_stream)
    out_lens = back[:4 * count].view(np.uint32)
    res = []
    for k, st in zip(out_lens, back[at_st:].view(np.uint64).reshape(count, 4)):
        code = int(st[0] & 0xFFFFFFFF)
        res.append((int(k), from_c(_lib.SbError(code, 0, int(st[1]), int(st[2]), int(st[3]))) if code else None))
    return res


def validate_batch(units) -> list:
    """Every unit checked as `Decoder().decompress_vec(unit)` would check it, without its decoded bytes: one
    sb_validate_batch_device_ws call on the current torch stream. Units are bytes-like; they go to the device in one
    copy and only out_lens and the statuses come back. Returns [(nbytes, error)]: the decoded length and None, or 0 and
    the error decompress_vec would raise (returned, not raised)."""
    import torch
    L = _lib.lib()

    def run(b, in_bytes, t_res, stream):
        need = L.sb_decompress_batch_scratch_bytes(b.count, in_bytes)
        t_scr = torch.empty(need, dtype=torch.uint8, device=t_res.device)
        e = _lib.SbError()
        if L.sb_validate_batch_device_ws(C.byref(b), in_bytes, None, t_scr.data_ptr(), need, stream, C.byref(e)):
            raise from_c(e)
        return t_res.cpu().numpy()

    return _validate_units(units, run)


def _stored_tables(tables, lens, dev, magic, rec, records):
    """Tables given to a reader: bytes-like ones go to the device in one copy, CUDA uint8 tensors are kept. Every header
    is checked on the host (size, magic, the stream length it was built over); records(words) is the record count a
    header announces. Returns (device tensors, headers as arrays of eight 64-bit words)."""
    import numpy as np
    import torch
    tables = list(tables)
    if len(tables) != len(lens):
        raise ValueError("%d tables for %d streams" % (len(tables), len(lens)))
    out, host = [], []
    for i, t in enumerate(tables):
        if isinstance(t, torch.Tensor):
            if not t.is_cuda or t.dtype != torch.uint8 or t.dim() != 1 or not t.is_contiguous() or t.data_ptr() % 8:
                raise ValueError("table %d: tables are bytes-like or contiguous 1-D 8-byte aligned CUDA uint8 tensors" % i)
            out.append(t)
        else:
            v = np.frombuffer(t, dtype=np.uint8)
            host.append((i, v))
            out.append(None)
    if host:                                                             # 8-byte multiples, so every table stays aligned
        at = np.cumsum([0] + [(v.size + 7) // 8 * 8 for _, v in host])
        cat = np.zeros(int(at[-1]) + 8, dtype=np.uint8)
        for (_, v), o in zip(host, at):
            cat[o:o + v.size] = v
        t_all = torch.from_numpy(cat).to(dev)
        for (i, v), o in zip(host, at):
            out[i] = t_all[int(o):int(o) + v.size]
    heads = {i: v[:64] for i, v in host if v.size >= 64}
    dev_heads = [i for i, t in enumerate(out) if i not in heads and t.numel() >= 64]
    if dev_heads:
        back = torch.stack([out[i][:64] for i in dev_heads]).cpu().numpy()
        heads.update(zip(dev_heads, back))
    words = []
    for i, (t, n) in enumerate(zip(out, lens)):
        if i not in heads:
            raise ValueError("table %d has %d bytes; a table has a 64-byte header" % (i, t.numel()))
        w = np.frombuffer(np.ascontiguousarray(heads[i]).tobytes(), dtype=np.uint64)
        if int(w[0]) != magic:
            raise ValueError("table %d is not a seek table of this format" % i)
        if int(w[1]) != n:
            raise ValueError("table %d was built over a stream of %d bytes; stream %d has %d" % (i, int(w[1]), i, n))
        if t.numel() < 64 + rec * records(w):
            raise ValueError("table %d has %d bytes; its header announces %d records" % (i, t.numel(), records(w)))
        words.append(w)
    return out, words


GATHER_RANGES_PER_CALL = 1 << 20            # ranges one gather call takes: its scratch is 108 bytes each plus 256 MiB
HOST_BUILD_BYTES = 1 << 30                  # compressed bytes a host-stream reader holds on the device to build tables


def _host_streams(streams):
    """The streams of a reader with host=True, as CPU uint8 tensors the device reads at their own addresses: bytes-like
    streams copied once into one pinned buffer, pinned 1-D contiguous CPU uint8 tensors as they are. Anything else
    raises ValueError before the library sees it; then every stream must pass sb_host_stream_check."""
    import numpy as np
    import torch
    out, host = [], []
    for i, s in enumerate(streams):
        if isinstance(s, torch.Tensor):
            if s.is_cuda or s.dtype != torch.uint8 or s.dim() != 1 or not s.is_contiguous() or not s.is_pinned():
                raise ValueError("stream %d: host=True takes bytes-like streams or pinned contiguous 1-D CPU uint8 "
                                 "tensors" % i)
            out.append(s)
        else:
            host.append((i, np.frombuffer(s, dtype=np.uint8)))
            out.append(None)
    if host:                                                             # the bytes-like streams in one pinned copy
        at = np.cumsum([0] + [v.size for _, v in host])
        t_all = torch.empty(int(at[-1]) + 1, dtype=torch.uint8, pin_memory=True)
        cat = t_all.numpy()
        for (i, v), o in zip(host, at):
            cat[o:o + v.size] = v
            out[i] = t_all[int(o):int(o) + v.size]
    L = _lib.lib()
    for t in out:
        e = _lib.SbError()
        if L.sb_host_stream_check(t.data_ptr(), t.numel(), C.byref(e)):
            raise from_c(e)
    return out


def _windows(which, lens, limit):
    """Groups of `which` whose lengths sum to at most `limit`; a longer stream makes a group of its own."""
    groups, cur, total = [], [], 0
    for i in which:
        if cur and total + lens[i] > limit:
            groups.append(cur)
            cur, total = [], 0
        cur.append(i)
        total += lens[i]
    if cur:
        groups.append(cur)
    return groups


def _check_ranges(ranges, count):
    """Ranges as (stream, lo, n) ints; IndexError or ValueError as read_ranges raises them."""
    ranges = [(int(i), int(lo), int(n)) for i, lo, n in ranges]
    for i, lo, n in ranges:
        if not 0 <= i < count:
            raise IndexError("stream %d of %d" % (i, count))
        if lo < 0 or n < 0 or lo + n > 0xFFFFFFFFFFFFFFFF:
            raise ValueError("range (%d, %d) is not within 64-bit offsets" % (lo, n))
    return ranges


def _gather(reader, fmt, ranges, rooms, data, offs):
    """sb_{fmt}_table_gather_device_ws over `ranges` (stream, lo, n) of a TableReader, each into data[offs[j]:] (rooms[j]
    bytes), in calls of at most GATHER_RANGES_PER_CALL ranges and BYTES_PER_CALL output bytes (a single larger range gets
    its own call). Returns the first failing range (its index in `ranges`) and its error, or None."""
    import numpy as np
    import torch
    L = _lib.lib()
    kind = "gather_host_streams" if reader._host else "gather"
    scratch_bytes = getattr(L, "sb_%s_table_%s_scratch_bytes" % (fmt, kind))
    call = getattr(L, "sb_%s_table_%s%s" % (fmt, kind, "_ws" if reader._host else "_device_ws"))
    a, k = 0, len(ranges)
    rooms = np.asarray(rooms, dtype=np.int64)
    ends = np.cumsum(rooms)
    while a < k:
        b = min(k, a + GATHER_RANGES_PER_CALL)
        base = int(ends[a - 1]) if a else 0
        b = max(a + 1, min(b, int(np.searchsorted(ends, base + reader.BYTES_PER_CALL, side="right"))))
        part = ranges[a:b]
        m = b - a
        desc = np.concatenate([np.array([lo for _, lo, _ in part] + [n for _, _, n in part], dtype=np.uint64).view(np.int64),
                               np.asarray(offs[a:b], dtype=np.int64) + data.data_ptr()])
        t_desc = torch.from_numpy(desc).to(reader._dev)
        t_unit = torch.from_numpy(np.array([i for i, _, _ in part] + [0], dtype=np.uint32).view(np.int32)).to(reader._dev)
        t_res = torch.zeros(5 * m, dtype=torch.int64, device=reader._dev)       # out_lens, statuses
        need = scratch_bytes(m)
        scr = torch.empty(need, dtype=torch.uint8, device=reader._dev)
        e = _lib.SbError()
        p = t_desc.data_ptr()
        if call(reader._t_tables.data_ptr(), reader._t_ins.data_ptr(), reader._t_lens.data_ptr(), len(reader._ins),
                t_unit.data_ptr(), p, p + 8 * m, p + 16 * m, t_res.data_ptr(), t_res.data_ptr() + 8 * m, m,
                scr.data_ptr(), need, reader._cuda, C.byref(e)):
            raise from_c(e)
        sts = t_res[m:].cpu().numpy().view(np.uint64).reshape(m, 4)
        bad = np.nonzero(sts[:, 0] & 0xFFFFFFFF)[0]
        if bad.size:
            s = sts[int(bad[0])]
            return a + int(bad[0]), from_c(_lib.SbError(int(s[0] & 0xFFFFFFFF), 0, int(s[1]), int(s[2]), int(s[3])))
        a = b
    return None


def _split(data, offs):
    """What gather returned, as read_ranges returns it: one bytes object per range."""
    back = data.cpu().numpy()
    return [back[int(a):int(b)].tobytes() for a, b in zip(offs[:-1], offs[1:])]


def _gathered(rooms):
    """The offsets of ranges packed back to back: len(rooms) + 1 int64 entries."""
    import numpy as np
    offs = np.zeros(len(rooms) + 1, dtype=np.int64)
    offs[1:] = np.cumsum(np.asarray(rooms, dtype=np.int64))
    return offs


class TableReader:
    """Random access to the decoded bytes of many raw streams on the device. Each stream gets a seek table, built once on
    the device in batch calls (sb_raw_table_build_batch_device_ws), one per group of streams whatever their number: the
    compressed offset and CRC of every 64 KiB output block, every block decoded and checksummed once. `read_ranges([(i,
    lo, n), ...])` then serves ranges of any of the streams in one library call per group, decoding and checksumming only
    the blocks they cover. Every range gives `Decoder().decompress_vec(streams[i])[lo:lo + n]`. A stream that is not
    seekable (see `seekable`: not block-independent, or not decodable) is decoded whole on the device for each call
    that reads it, and gives exactly that slice or raises that call's error. A stream is a bytes-like object (uploaded
    with the others in one copy) or a contiguous 1-D CUDA uint8 tensor (kept alive), of at most 2^32 - 1 bytes. Calls run
    on the current torch stream and wait for their results.
    tables: the streams' stored seek tables (from compress_batch(..., tables=True) or an earlier build), bytes-like or
    CUDA uint8 tensors, instead of a build. They are uploaded in one copy and no build runs; a table whose header does
    not match its stream's length raises ValueError. A table of another stream of the same length gives every read over
    it that block's checksum error, never wrong bytes.
    host: the streams stay in pinned host memory (bytes-like ones copied once into one pinned buffer, pinned CPU uint8
    tensors kept alive; unpinned CPU and CUDA tensors raise ValueError), so a corpus larger than the device can be read.
    Only the tables live on the device: they are built from uploads of at most HOST_BUILD_BYTES of streams at a time.
    Reads go through sb_raw_table_gather_host_streams_ws, which copies over PCIe only the compressed blocks it decodes;
    read_ranges is then the gather, split. Results and errors are those of a reader without host."""

    RANGES_PER_CALL = 4096                    # 128 KiB of staging per range: 512 MiB per call at most
    BYTES_PER_CALL = 1 << 30                  # output bytes one call gathers (a single larger range gets its own call)
    GROUP_BYTES = 1 << 34                     # compressed bytes one build call takes (its scratch grows with them)

    def __init__(self, streams, tables=None, host=False):
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
        for i, v in host:
            if v.size > 0xFFFFFFFF:
                raise ValueError("stream %d has %d bytes; a raw stream has at most 2^32 - 1" % (i, v.size))
        if host:                                                         # the bytes-like streams go up in one copy
            at = np.cumsum([0] + [v.size for _, v in host])
            cat = np.empty(int(at[-1]) + 1, dtype=np.uint8)
            for (_, v), o in zip(host, at):
                cat[o:o + v.size] = v
            t_all = torch.from_numpy(cat).to(self._dev)
            for (i, v), o in zip(host, at):
                self._ins[i] = t_all[int(o):int(o) + v.size]
        lens = [t.numel() for t in self._ins]
        for i, n in enumerate(lens):
            if n > 0xFFFFFFFF:
                raise ValueError("stream %d has %d bytes; a raw stream has at most 2^32 - 1" % (i, n))
        count = len(self._ins)
        self._bufs = []                                                  # the tables live in these
        if tables is not None:
            self._bufs, heads = _stored_tables(tables, lens, self._dev, _RAW_TABLE_MAGIC, 8,
                                               lambda w: int(w[3]) >> 32)
            ptrs = [t.data_ptr() for t in self._bufs]
            self.seekable = [int(w[4]) & 0xFFFFFFFF == 1 for w in heads]
            self.lengths = [int(w[2]) if ok else None for w, ok in zip(heads, self.seekable)]
        else:
            ptrs, results = [0] * count, [None] * count
            groups = _windows(range(count), lens, HOST_BUILD_BYTES) if self._host else [list(range(count))]
            for g in groups:                                             # host streams: one uploaded window at a time
                ins = {i: self._ins[i].to(self._dev) for i in g} if self._host else self._ins
                for i, p, r in self._build(g, ins):
                    ptrs[i], results[i] = p, r
                del ins
            self.seekable = [r.status.code == 0 for r in results]
            self.lengths = [int(r.bytes) if ok else None for r, ok in zip(results, self.seekable)]
        to64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).to(self._dev)
        self._t_tables = to64(ptrs + [0])
        self._t_ins = to64([t.data_ptr() for t in self._ins] + [0])
        self._t_lens = to64(lens + [0])

    def _build(self, which, streams):
        """sb_raw_table_build_batch_device_ws over groups of at most GROUP_BYTES compressed bytes of `streams` (device
        tensors by stream index): one call and one wait per group. A group's tables stay in one buffer cut to their
        packed size. Yields (stream, its table's address, its result) for every stream."""
        import numpy as np
        import torch
        L = _lib.lib()
        groups = _windows(which, [t.numel() if t is not None else 0 for t in self._ins], self.GROUP_BYTES)
        rsz = C.sizeof(_lib.SbFrameResult)
        for g in groups:
            k = len(g)
            ins = [streams[i] for i in g]
            in_bytes = sum(t.numel() for t in ins)
            desc = np.concatenate([np.array([t.data_ptr() for t in ins], dtype=np.uint64).view(np.int64),
                                   np.array([t.numel() for t in ins] + [0] * (k % 2), dtype=np.uint32).view(np.int64)])
            t_desc = torch.from_numpy(desc).to(self._dev)
            b = _lib.SbBatch()
            b.in_ptrs, b.in_lens, b.count = t_desc.data_ptr(), t_desc.data_ptr() + 8 * k, k
            tb = L.sb_raw_table_batch_bytes(k, in_bytes)
            t_tab = torch.empty(tb, dtype=torch.uint8, device=self._dev)
            t_res = torch.empty(8 * (k + 1) + rsz * k, dtype=torch.uint8, device=self._dev)   # offsets, then results
            need = L.sb_raw_table_build_batch_scratch_bytes(k, in_bytes)
            scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
            e = _lib.SbError()
            if L.sb_raw_table_build_batch_device_ws(C.byref(b), in_bytes, t_tab.data_ptr(), tb, t_res.data_ptr(),
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

    def __len__(self):
        return len(self._ins)

    def _call(self, ranges):
        """One sb_raw_table_decode_ranges_device_ws call: (out_lens, statuses, output tensor, offsets)."""
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
        need = L.sb_raw_table_ranges_scratch_bytes(k)
        scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
        e = _lib.SbError()
        p = t_desc.data_ptr()
        if L.sb_raw_table_decode_ranges_device_ws(self._t_tables.data_ptr(), self._t_ins.data_ptr(),
                                                  self._t_lens.data_ptr(), len(self._ins), t_unit.data_ptr(), p, p + 8 * k,
                                                  p + 16 * k, t_res.data_ptr(), t_res.data_ptr() + 8 * k, k,
                                                  scr.data_ptr(), need, self._cuda, C.byref(e)):
            raise from_c(e)
        back = t_res.cpu().numpy().view(np.uint64)
        return back[:k], back[k:5 * k].reshape(k, 4), t_out, offs

    def _decode_whole(self, which, device=False):
        """Streams that are not seekable, each as Decoder().decompress_vec gives it: {stream: bytes or the exception},
        the decodable ones in one sb_decompress_batch_device_ws call. device: the bytes as CUDA uint8 tensors."""
        import numpy as np
        import torch
        L = _lib.lib()
        got, todo = {}, []
        for i in which:
            try:                                                          # decompress_vec sizes its buffer this way
                todo.append((i, decompress_len(self._ins[i][:10].cpu().numpy().tobytes())))
            except Exception as x:
                got[i] = x
        if not todo:
            return got
        k = len(todo)
        caps = [dn for _, dn in todo]
        at = np.zeros(k, dtype=np.int64)
        at[1:] = np.cumsum(caps[:-1])
        t_out = torch.empty(sum(caps) + 1, dtype=torch.uint8, device=self._dev)
        ins = [self._ins[i].to(self._dev) for i, _ in todo]                # host streams: uploaded for this call
        desc = np.concatenate([np.array([t.data_ptr() for t in ins], dtype=np.uint64).view(np.int64), at + t_out.data_ptr(),
                               np.array([t.numel() for t in ins] + caps, dtype=np.uint32).view(np.int64)])
        t_desc = torch.from_numpy(desc).to(self._dev)
        t_res = torch.zeros(k + 4 * k, dtype=torch.int64, device=self._dev)   # out_lens (u32), statuses
        b = _lib.SbBatch()
        p = t_desc.data_ptr()
        b.in_ptrs, b.out_ptrs, b.in_lens, b.out_caps = p, p + 8 * k, p + 16 * k, p + 20 * k
        b.out_lens, b.statuses, b.count = t_res.data_ptr(), t_res.data_ptr() + 8 * k, k
        in_bytes = sum(t.numel() for t in ins)
        need = L.sb_decompress_batch_scratch_bytes(k, in_bytes)
        scr = torch.empty(need, dtype=torch.uint8, device=self._dev)
        e = _lib.SbError()
        if L.sb_decompress_batch_device_ws(C.byref(b), in_bytes, None, scr.data_ptr(), need, self._cuda, C.byref(e)):
            raise from_c(e)
        st = t_res.cpu().numpy().view(np.uint64)[k:].reshape(k, 4)
        back = t_out if device else t_out.cpu().numpy()
        for j, (i, dn) in enumerate(todo):
            s = st[j]
            got[i] = from_c(_lib.SbError(int(s[0] & 0xFFFFFFFF), 0, int(s[1]), int(s[2]), int(s[3]))) \
                if s[0] & 0xFFFFFFFF else back[at[j]:at[j] + dn] if device else back[at[j]:at[j] + dn].tobytes()
        return got

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
        whole = self._decode_whole(sorted({i for i, _, _ in ranges if not self.seekable[i]}))
        tabled = [r for r in ranges if self.seekable[r[0]]]
        got, a = [], 0
        while a < len(tabled):
            b, size = a, 0
            while b < len(tabled) and b - a < self.RANGES_PER_CALL:
                i, lo, n = tabled[b]
                room = max(0, min(n, self.lengths[i] - lo))
                if b > a and size + room > self.BYTES_PER_CALL:
                    break
                size += room
                b += 1
            lens, sts, t_out, offs = self._call(tabled[a:b])
            back = t_out.cpu().numpy()
            for s, o, m in zip(sts, offs, lens):
                got.append(from_c(_lib.SbError(int(s[0] & 0xFFFFFFFF), 0, int(s[1]), int(s[2]), int(s[3])))
                           if s[0] & 0xFFFFFFFF else back[o:o + int(m)].tobytes())
            a = b
        out, it = [], iter(got)
        for i, lo, n in ranges:
            r = next(it) if self.seekable[i] else whole[i]
            if isinstance(r, Exception):
                raise r
            out.append(r[lo:lo + n] if not self.seekable[i] else r)
        return out

    def gather(self, ranges):
        """Every (i, lo, n) range of stream i gathered on the device: (data, offsets), data one CUDA uint8 tensor with
        the ranges back to back and offsets an int64 array of len(ranges) + 1 entries, data[offsets[j]:offsets[j + 1]]
        being read_ranges(ranges)[j]. Ranges may be as read_ranges takes them; the ranges of seekable streams go through
        sb_raw_table_gather_device_ws, which decodes a block shared by many ranges as an edge once per call, in calls of
        up to GATHER_RANGES_PER_CALL ranges and BYTES_PER_CALL output bytes. A stream that is not seekable is decoded
        whole once and sliced on the device. Raises the first failing range's error, as read_ranges does."""
        import torch
        ranges = _check_ranges(ranges, len(self._ins))
        whole = self._decode_whole(sorted({i for i, _, _ in ranges if not self.seekable[i]}), device=True)
        rooms = []
        for i, lo, n in ranges:
            w = whole.get(i)
            size = w.numel() if isinstance(w, torch.Tensor) else self.lengths[i] if self.seekable[i] else 0
            rooms.append(max(0, min(n, size - lo)))
        offs = _gathered(rooms)
        data = torch.empty(int(offs[-1]), dtype=torch.uint8, device=self._dev)
        tabled = [j for j, (i, _, _) in enumerate(ranges) if self.seekable[i]]
        bad = _gather(self, "raw", [ranges[j] for j in tabled], [rooms[j] for j in tabled], data, offs[tabled]) \
            if tabled else None
        first, err = (tabled[bad[0]], bad[1]) if bad else (len(ranges), None)
        for j, (i, lo, n) in enumerate(ranges):
            if self.seekable[i]:
                continue
            if isinstance(whole[i], Exception):
                if j < first:
                    raise whole[i]
            elif rooms[j]:
                data[int(offs[j]):int(offs[j + 1])].copy_(whole[i][lo:lo + rooms[j]])
        if err is not None:
            raise err
        return data, offs

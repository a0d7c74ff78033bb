"""Tabled batch encodes on the GPU (sb_compress_batch_tabled_device_ws, sb_frame_encode_batch_tabled_device_ws,
raw.compress_batch, frame.encode_batch, TableReader(..., tables=)). Every output, out_len, status and chunk index must
equal the untabled call's; every table and result must be byte-identical to the batch build over the outputs
(sb_raw_table_build_batch_device_ws, sb_frame_table_build_batch_device_ws); nothing may be written past the tables, the
offsets, the results or the scratch; and readers over stored tables must read what readers over built tables read."""
import ctypes as C
import random

import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

BLOCK = 65536
MIB = 1 << 20
HEAD = 64
GUARD = 256
INVALID = 202
CORPUS = ("alice29.txt", "lcet10.txt", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata", "html_x_4",
          "paper-100k.pdf", "plrabn12.txt")


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _i64(v):
    import torch
    return torch.from_numpy(np.array(list(v), dtype=np.uint64).view(np.int64)).cuda()


def _u32(v):
    import torch
    return torch.from_numpy(np.array(list(v), dtype=np.uint32).view(np.int32)).cuda()


def frame_max_len(n):
    return 10 + (n + BLOCK - 1) // BLOCK * (8 + 76490)


class Source:
    """Unit inputs on the device: views at odd offsets into one text buffer, one random buffer and one zero buffer."""

    def __init__(self, nbytes, seed=0):
        import torch
        base = np.frombuffer(b"".join(corpus(c) for c in ("alice29.txt", "lcet10.txt", "html_x_4", "urls.10K")),
                             dtype=np.uint8).copy()
        reps = nbytes // base.size + 2
        self.text = torch.from_numpy(base).cuda().repeat(reps)
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.rand = torch.randint(0, 256, (nbytes + 64,), dtype=torch.uint8, device="cuda", generator=g)
        self.zero = torch.zeros(nbytes + 64, dtype=torch.uint8, device="cuda")
        self.base_size = base.size

    def view(self, kind, n, seed):
        at = 1 + 2 * (seed * 7919 % (self.base_size // 2))
        src = {"text": self.text, "rand": self.rand, "zero": self.zero}[kind]
        if kind != "text":
            at = 1 + 2 * (seed % 16)
        return src[at:at + n]


class Enc:
    """One batch encode over device inputs (tensors), untabled or tabled, with guard bytes after every output, the
    tables, the offsets, the results and the scratch."""

    def __init__(self, snap, ins, frame, caps=None, in_bytes=None, index=False):
        import torch
        self.snap, self.L, self.frame = snap, snap._lib.lib(), frame
        self.ins, self.n = ins, len(ins)
        lens = [t.numel() for t in ins]
        need = [frame_max_len(k) if frame else self.L.sb_max_compress_len(k) for k in lens]
        self.caps = need if caps is None else caps
        self.room = [min(c, 1 << 31) for c in self.caps]
        self.at = np.concatenate([[0], np.cumsum([r + GUARD for r in self.room[:-1]])]).astype(np.int64)
        self.in_bytes = sum(k for k, c, m in zip(lens, self.caps, need) if k > BLOCK and c >= m > 0) \
            if in_bytes is None else in_bytes
        self.t_ip = _i64([t.data_ptr() for t in ins] + [0])
        self.t_lens = _u32(lens + [0])
        self.t_caps = _u32(self.caps + [0])
        self.index = index
        self.nidx = sum((k + BLOCK - 1) // BLOCK + 1 for k in lens)
        self.t_tab_size = (self.L.sb_frame_encode_tables_bytes if frame else self.L.sb_compress_tables_bytes)(
            self.n, self.in_bytes)
        self.need_plain = (self.L.sb_frame_encode_batch_scratch_bytes if frame else self.L.sb_compress_batch_scratch_bytes)(
            self.n, self.in_bytes)
        self.need = (self.L.sb_frame_encode_batch_tabled_scratch_bytes if frame else
                     self.L.sb_compress_batch_tabled_scratch_bytes)(self.n, self.in_bytes)
        self.t_scr = torch.full((max(self.need, self.need_plain) + GUARD,), 0xCD, dtype=torch.uint8, device="cuda")

    def fresh(self):
        """New output, index, tables, offsets and results, filled with guard patterns."""
        import torch
        self.t_out = torch.full((int(self.at[-1]) + self.room[-1] + GUARD,), 0xEE, dtype=torch.uint8, device="cuda")
        self.t_op = _i64([self.t_out.data_ptr() + int(o) for o in self.at] + [0])
        self.t_ol = torch.full((self.n + 2,), -1, dtype=torch.int32, device="cuda")
        self.t_st = torch.full((32 * self.n + 32,), 0xA5, dtype=torch.uint8, device="cuda")
        self.t_idx = torch.full((self.nidx + 4,), -1, dtype=torch.int64, device="cuda")
        self.t_tab = torch.full((self.t_tab_size + GUARD,), 0xAB, dtype=torch.uint8, device="cuda")
        self.t_offs = torch.full((self.n + 2,), -1, dtype=torch.int64, device="cuda")
        self.t_res = torch.full((48 * self.n + 48,), 0xA5, dtype=torch.uint8, device="cuda")

    def batch(self):
        b = self.snap._lib.SbBatch()
        b.in_ptrs, b.out_ptrs, b.in_lens, b.out_caps = self.t_ip.data_ptr(), self.t_op.data_ptr(), self.t_lens.data_ptr(), \
            self.t_caps.data_ptr()
        b.out_lens, b.statuses, b.count = self.t_ol.data_ptr(), self.t_st.data_ptr(), self.n
        return b

    def call(self, tabled, b=None, stream=None, tables=True, offs=True, res=True, scr=True, tb=None, sb=None):
        import torch
        e = self.snap._lib.SbError()
        st = (stream or torch.cuda.current_stream()).cuda_stream
        b = C.byref(b or self.batch())
        idx = self.t_idx.data_ptr() if self.index else None
        if not tabled:
            if self.frame:
                return self.L.sb_frame_encode_batch_device_ws(b, self.in_bytes, idx, self.t_scr.data_ptr(), self.need_plain,
                                                              st, C.byref(e))
            return self.L.sb_compress_batch_device_ws(b, self.in_bytes, self.t_scr.data_ptr(), self.need_plain, st,
                                                      C.byref(e))
        args = (self.t_tab.data_ptr() if tables else None, self.t_tab_size if tb is None else tb,
                self.t_offs.data_ptr() if offs else None, self.t_res.data_ptr() if res else None,
                self.t_scr.data_ptr() if scr else None, self.need if sb is None else sb, st, C.byref(e))
        if self.frame:
            return self.L.sb_frame_encode_batch_tabled_device_ws(b, self.in_bytes, idx, *args)
        return self.L.sb_compress_batch_tabled_device_ws(b, self.in_bytes, *args)

    def run(self, tabled, stream=None):
        """Encode into fresh buffers; returns the device state to compare."""
        import torch
        self.fresh()
        assert self.call(tabled, stream=stream) == 0
        torch.cuda.synchronize()
        assert bool((self.t_scr[max(self.need, self.need_plain):] == 0xCD).all())
        ol = self.t_ol.cpu().numpy().view(np.uint32)
        assert ol[self.n] == 0xFFFFFFFF and (self.t_st[32 * self.n:].cpu().numpy() == 0xA5).all()
        ends = [int(o) + r for o, r in zip(self.at, self.room)]
        guards = torch.stack([self.t_out[e:e + 16] for e in ends])        # nothing written past any cap
        assert bool((guards == 0xEE).all())
        state = {"out": self.t_out.clone(), "ol": ol[:self.n].copy(), "st": self.t_st.cpu().numpy()[:32 * self.n].copy(),
                 "idx": self.t_idx.cpu().numpy().copy() if self.index else None}
        if tabled:
            offs = self.t_offs.cpu().numpy().view(np.uint64)
            assert offs[0] == 0 and offs[self.n + 1] == 0xFFFFFFFFFFFFFFFF and offs[self.n] <= self.t_tab_size
            tab = self.t_tab.cpu().numpy()
            assert (tab[int(offs[self.n]):] == 0xAB).all()
            res = self.t_res.cpu().numpy()
            assert (res[48 * self.n:] == 0xA5).all()
            state["tables"] = [tab[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(self.n)]
            state["res"] = [res[48 * i:48 * (i + 1)].tobytes() for i in range(self.n)]
        return state

    def build(self, state):
        """The batch build over this encode's outputs (still in self.t_out): (tables, results)."""
        import torch
        L = self.L
        b = self.snap._lib.SbBatch()
        t_lens = _u32(list(state["ol"]) + [0])
        b.in_ptrs, b.in_lens, b.count = self.t_op.data_ptr(), t_lens.data_ptr(), self.n
        total = int(state["ol"].astype(np.uint64).sum())
        e = self.snap._lib.SbError()
        st = torch.cuda.current_stream().cuda_stream
        t_offs = torch.zeros(self.n + 1, dtype=torch.int64, device="cuda")
        t_res = torch.zeros(48 * self.n, dtype=torch.uint8, device="cuda")
        if self.frame:
            mc = min(sum(int(k) // 1024 + 16 for k in state["ol"]), (1 << 22) - 2)
            tb = L.sb_frame_table_batch_bytes(self.n, mc)
            need = L.sb_frame_table_build_batch_scratch_bytes(self.n, total, mc)
            t_tab = torch.empty(tb, dtype=torch.uint8, device="cuda")
            scr = torch.empty(need, dtype=torch.uint8, device="cuda")
            assert L.sb_frame_table_build_batch_device_ws(C.byref(b), total, 0, None, None, mc, t_tab.data_ptr(), tb,
                                                          t_offs.data_ptr(), t_res.data_ptr(), scr.data_ptr(), need, st,
                                                          C.byref(e)) == 0
        else:
            tb = L.sb_raw_table_batch_bytes(self.n, total)
            need = L.sb_raw_table_build_batch_scratch_bytes(self.n, total)
            t_tab = torch.empty(tb, dtype=torch.uint8, device="cuda")
            scr = torch.empty(need, dtype=torch.uint8, device="cuda")
            assert L.sb_raw_table_build_batch_device_ws(C.byref(b), total, t_tab.data_ptr(), tb, t_offs.data_ptr(),
                                                        t_res.data_ptr(), scr.data_ptr(), need, st, C.byref(e)) == 0
        offs = t_offs.cpu().numpy().view(np.uint64)
        tab, res = t_tab.cpu().numpy(), t_res.cpu().numpy()
        return [tab[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(self.n)], \
            [res[48 * i:48 * (i + 1)].tobytes() for i in range(self.n)]


def check(snap, ins, frame, **kw):
    """Untabled and tabled encodes agree; the tables equal the build's. Returns the tabled state."""
    import torch
    enc = Enc(snap, ins, frame, **kw)
    plain = enc.run(False)
    got = enc.run(True)
    assert torch.equal(plain["out"], got["out"])
    assert (plain["ol"] == got["ol"]).all() and (plain["st"] == got["st"]).all()
    if enc.index:
        assert (plain["idx"] == got["idx"]).all()
    tables, results = enc.build(got)
    written = got["ol"] > 0
    if not frame:                                                        # the build marks every written stream seekable
        seek = [np.frombuffer(t[32:36], dtype=np.uint32)[0] == 1 for t in tables]
        assert all(s == w for s, w in zip(seek, written))
    for i in range(enc.n):
        assert got["tables"][i] == tables[i], (i, ins[i].numel())
        assert got["res"][i] == results[i], i
    del plain
    return enc, got


def corpus_ins():
    import torch
    datas = [corpus(c) for c in CORPUS] + [b"", b"x", corpus("alice29.txt")[:BLOCK - 1], corpus("lcet10.txt")[:BLOCK],
                                          corpus("lcet10.txt")[:BLOCK + 1]]
    return [torch.from_numpy(np.frombuffer(d + b"\0", dtype=np.uint8).copy()).cuda()[:len(d)] for d in datas]


@pytest.mark.parametrize("frame", [False, True])
def test_corpus(snap, frame):
    check(snap, corpus_ins(), frame, index=frame)


@pytest.mark.parametrize("frame", [False, True])
def test_1024_text_units_of_1mib(snap, frame):
    src = Source(1024 * (MIB + 64))
    check(snap, [src.view("text", MIB, i) for i in range(1024)], frame)


@pytest.mark.parametrize("frame", [False, True])
def test_64_units_of_16mib(snap, frame):
    src = Source(16 * MIB + 64, seed=3)
    kinds = ["text", "rand", "zero", "text"]
    check(snap, [src.view(kinds[i % 4], 16 * MIB - (i % 3) * 7, i) for i in range(64)], frame, index=frame)


@pytest.mark.parametrize("frame", [False, True])
def test_one_unit_of_1gib(snap, frame):
    src = Source(1 << 30)
    check(snap, [src.view("text", 1 << 30, 5)], frame)


def small_mixed(src, count, seed):
    rng = random.Random(seed)
    lens = [0, 1, BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK, 3 * BLOCK + 65535]
    lens += [rng.choice([rng.randrange(1, 4096), rng.randrange(1, 200000)]) for _ in range(count - len(lens))]
    return [src.view(rng.choice(["text", "text", "rand", "zero"]), n, i) for i, n in enumerate(lens)]


@pytest.mark.parametrize("frame", [False, True])
def test_10000_small_mixed_units(snap, frame):
    src = Source(4 * MIB)
    check(snap, small_mixed(src, 10000, 1), frame, index=frame)


@pytest.mark.parametrize("frame", [False, True])
def test_rejected_units_and_lengths_over_in_bytes(snap, frame):
    src = Source(4 * MIB)
    ins = [src.view("text", n, i) for i, n in enumerate((3 * BLOCK + 5, 500, 2 * BLOCK, BLOCK, 100))]
    need = [frame_max_len(t.numel()) if frame else snap._lib.lib().sb_max_compress_len(t.numel()) for t in ins]
    caps = need[:3] + [need[3] - 1, need[4]]                             # one cap a byte short: BufferTooSmall
    enc, got = check(snap, ins, frame, caps=caps)
    assert got["ol"][3] == 0
    _, got = check(snap, ins, frame, caps=need, in_bytes=5 * BLOCK + 4)  # the multi-block units past in_bytes
    assert got["ol"][0] == 0 and got["ol"][2] == 0 and got["ol"][1] > 0


@pytest.mark.parametrize("frame", [False, True])
def test_call_rules(snap, frame):
    """The same launches for 1 and 10,000 units; no allocation; short tables or scratch and null pointers launch
    nothing; a side stream behind pending work gives the same results."""
    import torch
    L = snap._lib.lib()
    src = Source(4 * MIB)
    one = Enc(snap, [src.view("text", 3 * BLOCK + 1, 1)], frame, index=frame)
    many = Enc(snap, small_mixed(src, 10000, 2), frame, index=frame)
    counts = []
    for e in (one, many):
        e.fresh()
        assert e.call(True) == 0                                         # warm up
        torch.cuda.synchronize()
        l0, a0 = L.sb_launch_count(), L.sb_alloc_count()
        assert e.call(True) == 0
        counts.append(L.sb_launch_count() - l0)
        assert L.sb_alloc_count() == a0
        e.fresh()
        l1 = L.sb_launch_count()
        assert e.call(False) == 0
        counts.append(L.sb_launch_count() - l1)
    assert counts[0] == counts[2] and counts[1] == counts[3] and counts[0] == counts[1] + 3
    l0 = L.sb_launch_count()
    for kw in ({"tables": False}, {"offs": False}, {"res": False}, {"scr": False}, {"tb": one.t_tab_size - 1},
               {"sb": one.need - 1}):
        assert one.call(True, **kw) == INVALID, kw
    b = one.batch()
    b.out_lens = None
    assert one.call(True, b=b) == INVALID
    b = one.batch()
    b.count = 1 << 31
    assert one.call(True, b=b) == INVALID
    b.count = 0
    assert one.call(True, b=b) == 0
    assert L.sb_launch_count() == l0
    # behind pending work: the input is written on the side stream just before the encode there
    data = src.view("text", 5 * MIB + 3, 4)
    ref = check(snap, [data], frame, index=frame)[1]
    dst = torch.zeros(data.numel() + 1, dtype=torch.uint8, device="cuda")[1:]
    side = torch.cuda.Stream()
    enc = Enc(snap, [dst], frame, index=frame)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        dst.copy_(data)
        got = enc.run(True, stream=side)
    assert torch.equal(got["out"][:int(got["ol"][0])], ref["out"][:int(ref["ol"][0])])
    assert got["tables"] == ref["tables"] and got["res"] == ref["res"]


def _units(seed):
    rng = random.Random(seed)
    text = b"".join(corpus(c) for c in ("alice29.txt", "lcet10.txt", "html_x_4"))
    out = [b"", b"a", text[:BLOCK], text[:3 * BLOCK + 17], bytes(2 * BLOCK + 1),
           np.random.default_rng(seed).integers(0, 256, BLOCK + 5, dtype=np.uint8).tobytes()]
    for _ in range(40):
        n = rng.randrange(0, 300000)
        k = rng.randrange(len(text) - n) if n < len(text) else 0
        out.append((text * 2)[k:k + n])
    return out


def test_python_batch_calls(snap):
    units = _units(1)
    enc = snap.raw.Encoder()
    streams = snap.raw.compress_batch(units)
    assert streams == [enc.compress_vec(u) for u in units]
    s2, tables = snap.raw.compress_batch(units, tables=True)
    assert s2 == streams and len(tables) == len(units)
    frames = snap.frame.encode_batch(units)
    assert frames == [snap.frame.encode_chunks(u, True) if u else b"" for u in units]
    f2, ftables = snap.frame.encode_batch(units, tables=True)
    assert f2 == frames and len(ftables) == len(units)


@pytest.mark.parametrize("frame", [False, True])
def test_table_reader_over_stored_tables(snap, frame):
    import torch
    L = snap._lib.lib()
    units = _units(2)
    mod = snap.frame if frame else snap.raw
    streams, tables = (snap.frame.encode_batch if frame else snap.raw.compress_batch)(units, tables=True)
    built = mod.TableReader(streams)
    stored = [bytes(bytearray(t)) for t in tables]                      # saved as bytes and reloaded
    torch.cuda.synchronize()
    l0 = L.sb_launch_count()
    reader = mod.TableReader(streams, tables=stored)
    assert L.sb_launch_count() == l0                                     # no build ran
    assert reader.lengths == built.lengths == [len(u) for u in units]
    if not frame:
        assert reader.seekable == built.seekable and all(reader.seekable)
    rng = random.Random(3)
    ranges = []
    for _ in range(4096):
        i = rng.randrange(len(units))
        ranges.append((i, rng.randrange(len(units[i]) + 1), rng.randrange(0, 70000)))
    assert reader.read_ranges(ranges) == built.read_ranges(ranges) == [units[i][lo:lo + n] for i, lo, n in ranges]
    # device tables work too
    dev = [torch.from_numpy(np.frombuffer(t, dtype=np.uint8).copy()).cuda() for t in tables]
    assert mod.TableReader(streams, tables=dev).read_ranges(ranges[:64]) == [units[i][lo:lo + n] for i, lo, n in ranges[:64]]
    # a table of a stream of another length
    with pytest.raises(ValueError, match="stream 3"):
        mod.TableReader(streams, tables=stored[:3] + [stored[4]] + stored[4:])
    # a table of another stream of the same length: the read's checksum error, never wrong bytes. Unit 5 is random,
    # so its first block is one literal (raw) or a stored chunk (frame): a byte changed there keeps the length
    other = bytearray(streams[5])
    other[100] ^= 0x55
    swapped = mod.TableReader([bytes(other)], tables=[tables[5]])
    if frame:
        with pytest.raises(snap.Error) as e:
            swapped.read(0, 0, len(units[5]))
        assert e.value.as_tuple()[0] == "Checksum"
    else:                                                                # Invalid{block, 0, 4}: a library-level status
        with pytest.raises(RuntimeError, match="code=202 a=0 b=0 c=4"):
            swapped.read(0, 0, len(units[5]))

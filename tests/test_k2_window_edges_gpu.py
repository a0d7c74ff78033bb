"""The window-edge streams of tests/test_k2_window_edges_emu.py on the H100: a replayed copy beside flattened ones,
more than 32 and more than 64 flattened copy bytes in one window, input spans loaded at their bound, streams shorter than
128 bytes, spans that reach past the stream's end and spills right after a new span, at each of the four input
alignments, and corrupted variants. Every unit's status, payload and bytes must be the oracle's: one warp per stream
(sb_decompress_batch_device), and through sb_decompress_batch_device_ws and the host batch."""
import pytest

import test_k2_window_edges_emu as edges
import test_legal_streams_emu as pop
from test_legal_streams_gpu import check_batches
from test_raw_batch_decode_gpu import Units

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _one_warp_per_stream(oracle, streams, caps, off):
    u = Units(streams, caps, off=off)
    rc, res, _, t_out = u.run(ws=False)
    assert rc == 0
    host_out = t_out.cpu().numpy()
    for i, (s, cap) in enumerate(zip(streams, caps)):
        want_st, want = pop._oracle(oracle, s, cap)
        assert res[i][0] == want_st, (off, i, res[i][0], want_st)
        if want is not None:
            o = u.ooffs[i]
            assert res[i][1] == len(want) and host_out[o:o + len(want)].tobytes() == want, (off, i)
        o = u.ooffs[i] + cap
        assert host_out[o:o + 16].tobytes() == b"\xee" * 16, (off, i)


def test_k2_window_edges_at_every_alignment(snap, oracle):
    ss, _ = edges.population()
    streams, caps = [s.stream for s in ss], [len(s.data) for s in ss]
    for off in range(4):
        _one_warp_per_stream(oracle, streams, caps, off)
    check_batches(snap, oracle, streams, caps)


def test_k2_corrupted_window_edges(snap, oracle):
    _, bad = edges.population()
    caps = [pop._header_cap(b) for b in bad]
    for off in range(4):
        _one_warp_per_stream(oracle, bad, caps, off)
    check_batches(snap, oracle, bad, caps)

"""K1 under a cap on chains per SM (SNAPB200_K1_CHAINS): same bytes as the oracle whatever the number of chains,
including caps that drop the L2-table chains or keep only some of them."""
import hashlib
import os
import subprocess
import sys

import pytest

from conftest import corpus
from kats import adversarial_blocks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# SNAPB200_K1_CHAINS / _NG are read once per process, hence one child process per setting
_CHILD = r"""
import hashlib, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import torch
torch.cuda.set_device(0)
import gpu_helpers
from test_k1_chain_cap import units
got = gpu_helpers.compress_batch_host(units())
print("DIGEST", len(got), hashlib.sha256(b"".join(len(g).to_bytes(4, "little") + g for g in got)).hexdigest())
"""


def distinct_units():
    us = adversarial_blocks()
    for name in ("alice29.txt", "html", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata"):
        d = corpus(name)
        us += [d[i:i + 65536] for i in range(0, len(d), 65536)]
    return us


def units():
    return distinct_units() * 30       # > 132 x 14 units: every SM runs as many chains as the cap allows


@pytest.mark.parametrize("chains,ng", [(1, 0), (5, 0), (3, 4), (9, 4)])
def test_k1_chain_cap(oracle, chains, ng):
    want = [oracle.compress(u) for u in distinct_units()] * 30
    digest = hashlib.sha256(b"".join(len(g).to_bytes(4, "little") + g for g in want)).hexdigest()
    env = dict(os.environ, SNAPB200_K1_CHAINS=str(chains), SNAPB200_K1_NG=str(ng))
    res = subprocess.run([sys.executable, "-c", _CHILD, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    line = [l for l in res.stdout.splitlines() if l.startswith("DIGEST")][-1].split()
    assert (int(line[1]), line[2]) == (len(want), digest)

import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DATA = os.path.join(ROOT, "tests", "golden", "data")

CORPUS = [
    "html", "urls.10K", "fireworks.jpeg", "paper-100k.pdf", "html_x_4",
    "alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt",
    "geo.protodata", "kppkn.gtb", "Mark.Twain-Tom.Sawyer.txt",
]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (H100, sm_90a)")


def corpus(name):
    with open(os.path.join(DATA, name), "rb") as f:
        return f.read()


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.lib()
    return o

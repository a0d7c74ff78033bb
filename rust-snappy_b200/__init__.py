"""rust-snappy_b200 -- host-side mirror of the `snap` crate's public API over
the C ABI of libsnapb200.so (hand-written sm_90a kernels; no CPU fallback).

    snap::raw::{Encoder, Decoder, max_compress_len, decompress_len} -> .raw
    snap::write::FrameEncoder                                      -> .write
    snap::read::{FrameDecoder, FrameEncoder}                       -> .read
    snap::Error                                                    -> .Error
"""
from . import _lib, frame, raw, read, shard, write  # noqa: F401
from .error import Error, NoDevice, UnexpectedEof  # noqa: F401

_lib.lib()  # fail loudly at import time when the CUDA library is not built

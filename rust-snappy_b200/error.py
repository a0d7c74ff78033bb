"""`snap::Error` mirrored as a Python exception (reference src/error.rs:72-186)."""

_VARIANTS = {
    1: ("TooBig", ("given", "max")),
    2: ("BufferTooSmall", ("given", "min")),
    3: ("Empty", ()),
    4: ("Header", ()),
    5: ("HeaderMismatch", ("expected_len", "got_len")),
    6: ("Literal", ("len", "src_len", "dst_len")),
    7: ("CopyRead", ("len", "src_len")),
    8: ("CopyWrite", ("len", "dst_len")),
    9: ("Offset", ("offset", "dst_pos")),
    10: ("StreamHeader", ("byte",)),
    11: ("StreamHeaderMismatch", ("bytes",)),
    12: ("UnsupportedChunkType", ("byte",)),
    13: ("UnsupportedChunkLength", ("len", "header")),
    14: ("Checksum", ("expected", "got")),
}


class Error(Exception):
    """One of the 14 `snap::Error` variants with its payload fields."""

    def __init__(self, variant, **fields):
        self.variant = variant
        self.fields = fields
        super().__init__("%s%s" % (variant, fields if fields else ""))

    def __eq__(self, other):
        return isinstance(other, Error) and (self.variant, self.fields) == (other.variant, other.fields)

    def __hash__(self):
        return hash((self.variant, tuple(sorted(self.fields.items()))))

    def as_tuple(self):
        """(variant, a, b, c) in the C ABI's payload order."""
        vals = list(self.fields.values())
        if self.variant == "StreamHeaderMismatch":
            vals = [int.from_bytes(self.fields["bytes"], "little")]
        if self.variant == "UnsupportedChunkLength":
            vals = [self.fields["len"], 1 if self.fields["header"] else 0]
        vals += [0] * (3 - len(vals))
        return (self.variant, vals[0], vals[1], vals[2])


class UnexpectedEof(EOFError):
    """io::ErrorKind::UnexpectedEof raised by read_exact (reference src/read.rs:439-455)."""


class NoDevice(RuntimeError):
    """The CUDA kernels cannot run here; this package has no CPU fallback."""


def from_c(e):
    code = e.code
    if code in _VARIANTS:
        name, fields = _VARIANTS[code]
        vals = [e.a, e.b, e.c]
        kw = dict(zip(fields, vals))
        if name == "StreamHeaderMismatch":
            kw = {"bytes": int(e.a).to_bytes(6, "little")}
        if name == "UnsupportedChunkLength":
            kw["header"] = bool(kw["header"])
        return Error(name, **kw)
    if code == 100:
        return UnexpectedEof("failed to fill whole buffer")
    if code == 200:
        return NoDevice("no usable CUDA device (sm_90a) for libsnapb200 -- there is no CPU fallback")
    return RuntimeError("libsnapb200 failure code=%d a=%d b=%d c=%d" % (code, e.a, e.b, e.c))

//! `snap` API surface (raw::{Encoder, Decoder, max_compress_len, decompress_len},
//! write::FrameEncoder, read::{FrameDecoder, FrameEncoder}, Error) forwarding the
//! hot path to the H100 kernels through the C ABI of include/snapb200.h.
//! Host code stays in Rust; nothing here compresses on the CPU.
use std::io;

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct SbError { pub code: u32, pub _pad: u32, pub a: u64, pub b: u64, pub c: u64 }

extern "C" {
    fn sb_max_compress_len(n: usize) -> usize;
    fn sb_compress(inp: *const u8, n: usize, out: *mut u8, cap: usize, out_n: *mut usize, e: *mut SbError) -> i32;
    fn sb_decompress_len(inp: *const u8, n: usize, out_len: *mut usize, e: *mut SbError) -> i32;
    fn sb_decompress(inp: *const u8, n: usize, out: *mut u8, cap: usize, out_n: *mut usize, e: *mut SbError) -> i32;
    fn sb_frame_max_len(n: usize) -> usize;
    fn sb_frame_encode_ex(inp: *const u8, n: usize, out: *mut u8, cap: usize, out_n: *mut usize, ident: i32, e: *mut SbError) -> i32;
    fn sb_frame_decode(inp: *const u8, n: usize, out: *mut u8, cap: usize, out_n: *mut usize, e: *mut SbError) -> i32;
}

/// Same variants and payload fields as the reference's `snap::Error`.
#[derive(Clone, Debug, PartialEq, Eq)]
pub enum Error {
    TooBig { given: u64, max: u64 }, BufferTooSmall { given: u64, min: u64 }, Empty, Header,
    HeaderMismatch { expected_len: u64, got_len: u64 }, Literal { len: u64, src_len: u64, dst_len: u64 },
    CopyRead { len: u64, src_len: u64 }, CopyWrite { len: u64, dst_len: u64 }, Offset { offset: u64, dst_pos: u64 },
    StreamHeader { byte: u8 }, StreamHeaderMismatch { bytes: Vec<u8> }, UnsupportedChunkType { byte: u8 },
    UnsupportedChunkLength { len: u64, header: bool }, Checksum { expected: u32, got: u32 },
    /// library-level failure (no device / CUDA error); never produced by the reference
    Device { code: u32, detail: u64 },
}
pub type Result<T> = std::result::Result<T, Error>;

/// Same messages as the reference (src/error.rs:249-335): callers match on them in logs and tests.
impl std::fmt::Display for Error {
    fn fmt(&self, f: &mut std::fmt::Formatter) -> std::fmt::Result {
        use Error::*;
        match self {
            TooBig { given, max } => write!(f, "snappy: input buffer (size = {}) is larger than allowed (size = {})", given, max),
            BufferTooSmall { given, min } => write!(f, "snappy: output buffer (size = {}) is smaller than required (size = {})", given, min),
            Empty => write!(f, "snappy: corrupt input (empty)"),
            Header => write!(f, "snappy: corrupt input (invalid header)"),
            HeaderMismatch { expected_len, got_len } => write!(f, "snappy: corrupt input (header mismatch; expected {} decompressed bytes but got {})", expected_len, got_len),
            Literal { len, src_len, dst_len } => write!(f, "snappy: corrupt input (expected literal read of length {}; remaining src: {}; remaining dst: {})", len, src_len, dst_len),
            CopyRead { len, src_len } => write!(f, "snappy: corrupt input (expected copy read of length {}; remaining src: {})", len, src_len),
            CopyWrite { len, dst_len } => write!(f, "snappy: corrupt input (expected copy write of length {}; remaining dst: {})", len, dst_len),
            Offset { offset, dst_pos } => write!(f, "snappy: corrupt input (expected valid offset but got offset {}; dst position: {})", offset, dst_pos),
            StreamHeader { byte } => write!(f, "snappy: corrupt input (expected stream header but got unexpected chunk type byte {})", byte),
            StreamHeaderMismatch { bytes } => {
                let esc: String = bytes.iter().flat_map(|&b| std::ascii::escape_default(b)).map(|b| b as char).collect();
                write!(f, "snappy: corrupt input (expected sNaPpY stream header but got {})", esc)
            }
            UnsupportedChunkType { byte } => write!(f, "snappy: corrupt input (unsupported chunk type: {})", byte),
            UnsupportedChunkLength { len, header: false } => write!(f, "snappy: corrupt input (unsupported chunk length: {})", len),
            UnsupportedChunkLength { len, header: true } => write!(f, "snappy: corrupt input (invalid stream header length: {})", len),
            Checksum { expected, got } => write!(f, "snappy: corrupt input (bad checksum; expected: {}, got: {})", expected, got),
            Device { code, detail } => write!(f, "snapb200: device failure (code {}, detail {})", code, detail),
        }
    }
}

/// `into_inner` of a writer failed to flush: carries the writer back together with the error (src/error.rs:15-60).
pub struct IntoInnerError<W> { wtr: W, err: io::Error }
impl<W> IntoInnerError<W> {
    pub fn error(&self) -> &io::Error { &self.err }
    pub fn into_error(self) -> io::Error { self.err }
    pub fn into_inner(self) -> W { self.wtr }
}
impl<W: std::any::Any> std::error::Error for IntoInnerError<W> {}
impl<W> std::fmt::Display for IntoInnerError<W> { fn fmt(&self, f: &mut std::fmt::Formatter) -> std::fmt::Result { self.err.fmt(f) } }
impl<W> std::fmt::Debug for IntoInnerError<W> { fn fmt(&self, f: &mut std::fmt::Formatter) -> std::fmt::Result { self.err.fmt(f) } }
impl std::error::Error for Error {}
impl From<Error> for io::Error { fn from(e: Error) -> io::Error { io::Error::new(io::ErrorKind::Other, e) } }

fn to_err(e: SbError) -> Error {
    match e.code {
        1 => Error::TooBig { given: e.a, max: e.b }, 2 => Error::BufferTooSmall { given: e.a, min: e.b },
        3 => Error::Empty, 4 => Error::Header, 5 => Error::HeaderMismatch { expected_len: e.a, got_len: e.b },
        6 => Error::Literal { len: e.a, src_len: e.b, dst_len: e.c }, 7 => Error::CopyRead { len: e.a, src_len: e.b },
        8 => Error::CopyWrite { len: e.a, dst_len: e.b }, 9 => Error::Offset { offset: e.a, dst_pos: e.b },
        10 => Error::StreamHeader { byte: e.a as u8 },
        11 => Error::StreamHeaderMismatch { bytes: e.a.to_le_bytes()[..6].to_vec() },
        12 => Error::UnsupportedChunkType { byte: e.a as u8 },
        13 => Error::UnsupportedChunkLength { len: e.a, header: e.b != 0 },
        14 => Error::Checksum { expected: e.a as u32, got: e.b as u32 },
        c => Error::Device { code: c, detail: e.a },
    }
}

pub mod raw {
    use super::*;
    pub fn max_compress_len(n: usize) -> usize { unsafe { sb_max_compress_len(n) } }
    pub fn decompress_len(input: &[u8]) -> Result<usize> {
        let (mut n, mut e) = (0usize, SbError::default());
        if unsafe { sb_decompress_len(input.as_ptr(), input.len(), &mut n, &mut e) } != 0 { return Err(to_err(e)); }
        Ok(n)
    }
    #[derive(Debug, Default)] pub struct Encoder { _p: () }
    impl Encoder {
        pub fn new() -> Encoder { Encoder { _p: () } }
        pub fn compress(&mut self, input: &[u8], output: &mut [u8]) -> Result<usize> {
            let (mut n, mut e) = (0usize, SbError::default());
            let rc = unsafe { sb_compress(input.as_ptr(), input.len(), output.as_mut_ptr(), output.len(), &mut n, &mut e) };
            if rc != 0 { Err(to_err(e)) } else { Ok(n) }
        }
        pub fn compress_vec(&mut self, input: &[u8]) -> Result<Vec<u8>> {
            let mut buf = vec![0; max_compress_len(input.len())];
            let n = self.compress(input, &mut buf)?;
            buf.truncate(n);
            Ok(buf)
        }
    }
    #[derive(Clone, Debug, Default)] pub struct Decoder { _p: () }
    impl Decoder {
        pub fn new() -> Decoder { Decoder { _p: () } }
        pub fn decompress(&mut self, input: &[u8], output: &mut [u8]) -> Result<usize> {
            let (mut n, mut e) = (0usize, SbError::default());
            let rc = unsafe { sb_decompress(input.as_ptr(), input.len(), output.as_mut_ptr(), output.len(), &mut n, &mut e) };
            if rc != 0 { Err(to_err(e)) } else { Ok(n) }
        }
        pub fn decompress_vec(&mut self, input: &[u8]) -> Result<Vec<u8>> {
            let mut buf = vec![0; decompress_len(input)?];
            let n = self.decompress(input, &mut buf)?;
            buf.truncate(n);
            Ok(buf)
        }
    }
}

const MAX_BLOCK_SIZE: usize = 1 << 16;
const MAX_COMPRESS_BLOCK_SIZE: usize = 76490;   // src/frame.rs:12
const STREAM_IDENTIFIER: &[u8] = b"\xFF\x06\x00\x00sNaPpY";

fn encode_chunks(buf: &[u8], ident: bool) -> Result<Vec<u8>> {
    let cap = unsafe { sb_frame_max_len(buf.len()) };
    let mut out = vec![0u8; cap];
    let (mut n, mut e) = (0usize, SbError::default());
    let rc = unsafe { sb_frame_encode_ex(buf.as_ptr(), buf.len(), out.as_mut_ptr(), cap, &mut n, ident as i32, &mut e) };
    if rc != 0 { return Err(to_err(e)); }
    out.truncate(n);
    Ok(out)
}

pub mod write {
    use super::*;
    /// Same staging rules as the reference (src/write.rs:123-161): they fix the chunk boundaries.
    /// `with_batch(n)` queues up to n full 64KB chunks and encodes them with one device call; a partial chunk,
    /// flush(), into_inner() and drop drain the queue. The bytes written are the same, only later.
    pub struct FrameEncoder<W: io::Write> { w: Option<W>, src: Vec<u8>, queue: Vec<u8>, batch: usize, wrote_stream_ident: bool }
    impl<W: io::Write> FrameEncoder<W> {
        pub fn new(wtr: W) -> Self { Self::with_batch(wtr, 1) }
        pub fn with_batch(wtr: W, chunks: usize) -> Self {
            FrameEncoder { w: Some(wtr), src: Vec::with_capacity(MAX_BLOCK_SIZE), queue: Vec::new(), batch: chunks.max(1), wrote_stream_ident: false }
        }
        pub fn get_ref(&self) -> &W { self.w.as_ref().unwrap() }
        pub fn get_mut(&mut self) -> &mut W { self.w.as_mut().unwrap() }
        /// src/write.rs:91-96: a failed flush hands the encoder back inside the error.
        pub fn into_inner(mut self) -> std::result::Result<W, IntoInnerError<FrameEncoder<W>>> {
            match io::Write::flush(&mut self) {
                Ok(()) => Ok(self.w.take().unwrap()),
                Err(err) => Err(IntoInnerError { wtr: self, err }),
            }
        }
        fn drain(&mut self) -> io::Result<()> {
            if self.queue.is_empty() { return Ok(()); }
            let out = encode_chunks(&self.queue, false)?;
            self.queue.clear();
            self.w.as_mut().unwrap().write_all(&out)
        }
        fn inner_write(&mut self, buf: &[u8]) -> io::Result<usize> {
            if !self.wrote_stream_ident { self.wrote_stream_ident = true; self.w.as_mut().unwrap().write_all(STREAM_IDENTIFIER)?; }
            if buf.is_empty() { return Ok(0); }
            if self.batch == 1 { let out = encode_chunks(buf, false)?; self.w.as_mut().unwrap().write_all(&out)?; return Ok(buf.len()); }
            // chunk boundaries inside `buf` are every 64KB with the partial chunk last, so queued full chunks + buf
            // encode to the same bytes in one call as chunk by chunk
            self.queue.extend_from_slice(buf);
            if buf.len() % MAX_BLOCK_SIZE != 0 || self.queue.len() >= self.batch * MAX_BLOCK_SIZE { self.drain()?; }
            Ok(buf.len())
        }
    }
    impl<W: io::Write> io::Write for FrameEncoder<W> {
        fn write(&mut self, mut buf: &[u8]) -> io::Result<usize> {
            let mut total = 0;
            loop {
                let free = MAX_BLOCK_SIZE - self.src.len();
                let n = if buf.len() <= free { break } else if self.src.is_empty() { self.inner_write(buf)? } else {
                    self.src.extend_from_slice(&buf[..free]); self.flush_src()?; free };
                buf = &buf[n..]; total += n;
            }
            self.src.extend_from_slice(buf);
            Ok(total + buf.len())
        }
        fn flush(&mut self) -> io::Result<()> { self.flush_src()?; self.drain() }
    }
    impl<W: io::Write> FrameEncoder<W> {
        fn flush_src(&mut self) -> io::Result<()> {
            if self.src.is_empty() { return Ok(()); }
            let src = std::mem::take(&mut self.src);
            let r = self.inner_write(&src);
            self.src = src; self.src.clear();
            r.map(|_| ())
        }
    }
    impl<W: io::Write> Drop for FrameEncoder<W> { fn drop(&mut self) { if self.w.is_some() { let _ = io::Write::flush(self); } } }
}

pub mod read {
    use super::*;
    /// The reference's chunk state machine (src/read.rs:104-239): every refill pulls exactly the bytes of the next
    /// chunk(s) from the reader -- one data chunk with `new`, up to n with `with_batch(n)` (read-ahead; one device call
    /// per refill) -- and hands them to the device decoder (header walk, K2, checksum). Bytes decoded before a
    /// failing chunk are served first, then the error, like the reference.
    pub struct FrameDecoder<R: io::Read> { r: R, out: Vec<u8>, at: usize, batch: usize, seen_ident: bool, eof: bool, pending: Option<io::Error> }
    fn read_upto<R: io::Read>(r: &mut R, buf: &mut [u8]) -> io::Result<usize> {
        let mut k = 0;
        while k < buf.len() {
            match r.read(&mut buf[k..]) { Ok(0) => break, Ok(n) => k += n,
                Err(ref e) if e.kind() == io::ErrorKind::Interrupted => {}, Err(e) => return Err(e) }
        }
        Ok(k)
    }
    impl<R: io::Read> FrameDecoder<R> {
        pub fn new(rdr: R) -> Self { Self::with_batch(rdr, 1) }
        pub fn with_batch(rdr: R, chunks: usize) -> Self {
            FrameDecoder { r: rdr, out: vec![], at: 0, batch: chunks.max(1), seen_ident: false, eof: false, pending: None }
        }
        pub fn get_ref(&self) -> &R { &self.r }
        pub fn get_mut(&mut self) -> &mut R { &mut self.r }
        pub fn into_inner(self) -> R { self.r }
        fn refill(&mut self) -> io::Result<()> {
            // an identifier chunk in front stands in for the one already consumed (identifier chunks may repeat, :166-178)
            let mut raw: Vec<u8> = if self.seen_ident { STREAM_IDENTIFIER.to_vec() } else { vec![] };
            let base = raw.len();
            let mut chunks = 0;
            while chunks < self.batch && !self.eof {
                let mut head = [0u8; 4];
                let k = read_upto(&mut self.r, &mut head)?;
                raw.extend_from_slice(&head[..k]);
                if k < 4 { self.eof = true; break; }
                self.seen_ident = true;
                let len = head[1] as usize | (head[2] as usize) << 8 | (head[3] as usize) << 16;
                if len > MAX_COMPRESS_BLOCK_SIZE || (0x02..=0x7F).contains(&head[0]) { self.eof = true; break; }
                let at = raw.len();
                raw.resize(at + len, 0);
                let k = read_upto(&mut self.r, &mut raw[at..])?;
                raw.truncate(at + k);
                if k < len { self.eof = true; break; }
                if head[0] <= 0x01 { chunks += 1; }
            }
            self.out.clear(); self.at = 0;
            if raw.len() == base { return Ok(()); }
            let (mut n, mut e) = (0usize, SbError::default());
            if unsafe { sb_frame_decode(raw.as_ptr(), raw.len(), std::ptr::null_mut(), 0, &mut n, &mut e) } != 0 { self.pending = Some(to_io(e)); return Ok(()); }
            self.out.resize(n.max(1), 0);
            let rc = unsafe { sb_frame_decode(raw.as_ptr(), raw.len(), self.out.as_mut_ptr(), n, &mut n, &mut e) };
            self.out.truncate(n);
            if rc != 0 { self.pending = Some(to_io(e)); }
            Ok(())
        }
    }
    fn to_io(e: SbError) -> io::Error {
        if e.code == 100 { io::Error::new(io::ErrorKind::UnexpectedEof, "failed to fill whole buffer") } else { to_err(e).into() }
    }
    impl<R: io::Read> io::Read for FrameDecoder<R> {
        fn read(&mut self, buf: &mut [u8]) -> io::Result<usize> {
            if buf.is_empty() { return Ok(0); }
            loop {
                if self.at < self.out.len() {
                    let k = buf.len().min(self.out.len() - self.at);
                    buf[..k].copy_from_slice(&self.out[self.at..self.at + k]); self.at += k;
                    return Ok(k);
                }
                if let Some(e) = self.pending.take() { return Err(e); }
                if self.eof { return Ok(0); }
                self.refill()?;
            }
        }
    }
    /// One chunk per underlying read() of <=64KB (src/read.rs:368-409).
    pub struct FrameEncoder<R: io::Read> { r: R, src: Vec<u8>, dst: Vec<u8>, at: usize, wrote_stream_ident: bool }
    impl<R: io::Read> FrameEncoder<R> {
        pub fn new(rdr: R) -> Self { FrameEncoder { r: rdr, src: vec![0; MAX_BLOCK_SIZE], dst: vec![], at: 0, wrote_stream_ident: false } }
        pub fn get_ref(&self) -> &R { &self.r }
        pub fn get_mut(&mut self) -> &mut R { &mut self.r }
    }
    impl<R: io::Read> io::Read for FrameEncoder<R> {
        fn read(&mut self, buf: &mut [u8]) -> io::Result<usize> {
            if self.at >= self.dst.len() {
                let n = self.r.read(&mut self.src)?;
                if n == 0 { return Ok(0); }
                self.dst = encode_chunks(&self.src[..n], !self.wrote_stream_ident)?; self.wrote_stream_ident = true; self.at = 0;
            }
            let k = buf.len().min(self.dst.len() - self.at);
            buf[..k].copy_from_slice(&self.dst[self.at..self.at + k]); self.at += k;
            Ok(k)
        }
    }
}

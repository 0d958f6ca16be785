//! cuda_decoder — `flowgger::decoder::Decoder` implementations backed by the H100 batched parser.
//!
//! Mirrors flowgger_b200/csrc/host/flowgger.{hpp,cpp} (the C++ twin that the test-suite drives, because the
//! build environment has no Rust toolchain).  Reference interfaces implemented here:
//!   * `Decoder::decode(&self, line: &str) -> Result<Record, &'static str>`  (src/flowgger/decoder/mod.rs:44-46)
//!   * `CloneBoxedDecoder` via `#[derive(Clone)]`                            (decoder/mod.rs:23-42)
//!   * `Splitter<T>::run`                                                    (src/flowgger/splitter/mod.rs:18-26)
//! All parsing happens on the GPU — including line framing, the UTF-8 check and the unescape of RFC5424 SD values; this
//! crate hands raw blocks to `fg_split_decode` (or packed lines to `fg_decode_batch`) and materialises Records, or, for
//! the rfc5424 -> gelf and rfc3164 -> gelf pairs, forwards the records the device already framed, decoded and encoded
//! (`fg_split_decode_encode_gelf`).
#![allow(non_camel_case_types, non_upper_case_globals, dead_code)]

use flowgger::flowgger::config::Config;
use flowgger::flowgger::decoder::Decoder;
use flowgger::flowgger::encoder::{build_prepend_ts, config_get_prepend_ts, Encoder};
use flowgger::flowgger::record::{Record, SDValue, StructuredData};
use flowgger::flowgger::splitter::Splitter;
use std::ffi::{CStr, CString};
use std::io::{stderr, BufRead, BufReader, ErrorKind, Read, Write};
use std::os::raw::c_char;
use std::ptr;
use std::sync::mpsc::SyncSender;
use std::sync::{Arc, Mutex};

mod ffi {
    include!(concat!(env!("OUT_DIR"), "/ffi.rs"));
}
use ffi::*;

/// What `fg_create` was given apart from the capacity, kept to make a twin of a context with another capacity.
#[derive(Clone)]
struct CtxSpec {
    device: i32,
    has_schema: bool,
    names: Vec<CString>,
    types: Vec<i32>,
    suffix: [Option<String>; 5],
    tzdir: Option<CString>,
}

/// One GPU context of a fixed format (`fg_ctx`); shared by the clones handed to input threads.
struct Ctx {
    raw: *mut fg_ctx,
    fmt: fg_format,
    suffix: [Option<String>; 5],
    spec: CtxSpec,
    max_bytes: usize,                        // max_batch_bytes as fg_create took it
    extra: [Option<Vec<(String, String)>>; 3],  // the output.gelf_extra / ltsv_extra / capnp_extra last set on the context
}
unsafe impl Send for Ctx {}
impl Drop for Ctx {
    fn drop(&mut self) {
        unsafe { fg_destroy(self.raw) }
    }
}

#[derive(Clone)]
pub struct CudaDecoder {
    ctx: Arc<Mutex<Ctx>>,
}

fn ltsv_type(t: &str) -> Option<i32> {
    match t.to_lowercase().as_ref() {
        "string" => Some(0),
        "bool" => Some(1),
        "f64" => Some(2),
        "i64" => Some(3),
        "u64" => Some(4),
        _ => None,
    }
}

impl CudaDecoder {
    /// `RFC5424Decoder::new(&Config)` / `LTSVDecoder::new` / `GelfDecoder::new` / `RFC3164Decoder::new` replacement,
    /// selected in `flowgger::start` (src/flowgger/mod.rs:413-422) by `input.format`.
    /// RFC3164 (`fg_format_FG_FMT_RFC3164`): the context follows the UTC clock for `now_utc().year()`
    /// (rfc3164_decoder.rs:175, `rfc3164_year = 0`) and reads the zone database behind `timezones::get_by_name` (:196) from
    /// the TZif files under `input.cuda_tzdir` / `$TZDIR` / /usr/share/zoneinfo.
    pub fn new(config: &Config, fmt: fg_format) -> CudaDecoder {
        let mut names: Vec<CString> = Vec::new();
        let mut types: Vec<i32> = Vec::new();
        let mut suffix: [Option<String>; 5] = Default::default();
        let has_schema = config.lookup("input.ltsv_schema").is_some();
        if let Some(pairs) = config.lookup("input.ltsv_schema") {
            // same panics as ltsv_decoder.rs:31-44
            for (name, sdtype) in pairs.as_table().expect("input.ltsv_schema must be a list of key/type pairs") {
                let t = sdtype.as_str().expect("input.ltsv_schema types must be strings");
                let t = ltsv_type(t).unwrap_or_else(|| panic!("Unsupported type in input.ltsv_schema for name [{}]", name));
                names.push(CString::new(name.as_str()).unwrap());
                types.push(t);
            }
        }
        if let Some(pairs) = config.lookup("input.ltsv_suffixes") {
            for (sdtype, sfx) in pairs.as_table().expect("input.ltsv_suffixes must be a list of type/suffixes pairs") {
                let sfx = sfx.as_str().expect("input.ltsv_suffixes suffixes must be strings").to_owned();
                match ltsv_type(sdtype) {
                    Some(0) => panic!("Strings cannot be suffixed"),
                    Some(t) => suffix[t as usize] = Some(sfx),
                    None => panic!("Unsupported type in input.ltsv_suffixes for type [{}]", sdtype),
                }
            }
        }
        let spec = CtxSpec {
            device: config.lookup("input.cuda_device").and_then(|v| v.as_integer()).unwrap_or(0) as i32,
            has_schema,
            names,
            types,
            suffix,
            tzdir: config.lookup("input.cuda_tzdir").and_then(|v| v.as_str()).map(|s| CString::new(s).unwrap()),
        };
        let max_bytes = config.lookup("input.cuda_max_batch_bytes").and_then(|v| v.as_integer()).unwrap_or(0);
        let max_lines = config.lookup("input.cuda_max_batch_lines").and_then(|v| v.as_integer()).unwrap_or(0) as i32;
        CudaDecoder::create(spec, fmt, max_bytes, max_lines)
    }

    fn create(spec: CtxSpec, fmt: fg_format, max_bytes: i64, max_lines: i32) -> CudaDecoder {
        let name_ptrs: Vec<*const c_char> = spec.names.iter().map(|s| s.as_ptr()).collect();
        let sfx_c: Vec<Option<CString>> = spec.suffix.iter().map(|s| s.as_ref().map(|x| CString::new(x.as_str()).unwrap())).collect();
        let mut cfg: fg_config = unsafe { std::mem::zeroed() };
        cfg.device = spec.device;
        cfg.max_batch_bytes = max_bytes;
        cfg.max_batch_lines = max_lines;
        cfg.rfc3164_year = 0;
        cfg.tzdir = spec.tzdir.as_ref().map_or(ptr::null(), |s| s.as_ptr());
        cfg.input_format = fmt as i32;
        cfg.ltsv_has_schema = spec.has_schema as i32;
        cfg.ltsv_schema_len = spec.names.len() as i32;
        cfg.ltsv_schema_names = name_ptrs.as_ptr();
        cfg.ltsv_schema_types = spec.types.as_ptr();
        for t in 1..5 {
            cfg.ltsv_suffix[t] = sfx_c[t].as_ref().map_or(ptr::null(), |s| s.as_ptr());
        }
        let mut raw: *mut fg_ctx = ptr::null_mut();
        let rc = unsafe { fg_create(&cfg, &mut raw) };
        if rc != 0 {
            // There is no CPU fallback: without the library + a GPU the decoder cannot exist.
            panic!("flowgger_cuda: fg_create failed ({})", rc);
        }
        let max_bytes = if max_bytes > 0 { (max_bytes as usize).min(0x7FFF_FFC0) } else { 256 << 20 };  // fg_create's default and cap
        let suffix = spec.suffix.clone();
        CudaDecoder { ctx: Arc::new(Mutex::new(Ctx { raw, fmt, suffix, spec, max_bytes, extra: [None, None, None] })) }
    }

    /// max_batch_bytes of the context
    pub fn capacity_bytes(&self) -> usize {
        self.ctx.lock().unwrap().max_bytes
    }

    /// A context of the same format and configuration sized for `max_bytes` (one line longer than a whole batch).
    pub fn make_sized(&self, max_bytes: usize) -> CudaDecoder {
        let (spec, fmt) = {
            let c = self.ctx.lock().unwrap();
            (c.spec.clone(), c.fmt)
        };
        CudaDecoder::create(spec, fmt, max_bytes as i64, 64)
    }

    /// Decode `n` lines packed as bytes + offsets; calls `f(i, result)` in input order.
    pub fn decode_batch<F: FnMut(usize, Result<Record, &'static str>, &[String])>(&self, bytes: &[u8], offsets: &[i32], mut f: F) {
        let ctx = self.ctx.lock().unwrap();
        let n = offsets.len() - 1;
        let mut out: fg_batch_out = unsafe { std::mem::zeroed() };
        let rc = unsafe { fg_decode_batch(ctx.raw, ctx.fmt, bytes.as_ptr(), offsets.as_ptr(), n as i32, &mut out) };
        if rc != 0 {
            let e = unsafe { CStr::from_ptr(fg_last_error(ctx.raw)) }.to_string_lossy().into_owned();
            panic!("fg_decode_batch: {}", e);
        }
        for i in 0..n {
            let mut side = Vec::new();
            let r = materialize(&ctx, &out, bytes, offsets, i, &mut side);
            f(i, r, &side);
        }
    }
}

/// Extent of line i of a raw stream framed on the device without its terminator (BufRead::lines: the '\n' and one '\r'
/// before it)
fn line_extent(stream: &[u8], line_offsets: &[i32], i: usize) -> (usize, usize) {
    let (lo, mut hi) = (line_offsets[i] as usize, line_offsets[i + 1] as usize);
    if hi > lo && stream[hi - 1] == b'\n' { hi -= 1; if hi > lo && stream[hi - 1] == b'\r' { hi -= 1; } }
    (lo, hi)
}

/// The reference's `&'static str` for a status
fn error_str(fmt: fg_format, status: u32) -> &'static str {
    unsafe {
        let s = CStr::from_ptr(fg_error_string(fmt, status));
        std::str::from_utf8_unchecked(std::slice::from_raw_parts(s.as_ptr() as *const u8, s.to_bytes().len()))
    }
}

impl CudaDecoder {
    /// Framing + UTF-8 validation + decode of a raw stream on the device (`fg_split_decode`): `f(i, line, result)` in
    /// stream order; a line that is not UTF-8 arrives as `Err("Invalid UTF-8 input")` (line_splitter.rs:22-25).
    /// false (nothing decoded) when the stream does not fit the context: more bytes or more lines than it holds.
    pub fn split_decode<F: FnMut(usize, &[u8], Result<Record, &'static str>, &[String])>(&self, stream: &[u8], mut f: F) -> bool {
        let ctx = self.ctx.lock().unwrap();
        let mut out: fg_batch_out = unsafe { std::mem::zeroed() };
        let rc = unsafe { fg_split_decode(ctx.raw, ctx.fmt, stream.as_ptr(), stream.len() as i64, &mut out) };
        if rc == FG_E_CAPACITY {
            return false;
        }
        if rc != 0 {
            let e = unsafe { CStr::from_ptr(fg_last_error(ctx.raw)) }.to_string_lossy().into_owned();
            panic!("fg_split_decode: {}", e);
        }
        let offs = unsafe { std::slice::from_raw_parts(out.line_offsets, out.n as usize + 1) };
        for i in 0..out.n as usize {
            let (lo, hi) = line_extent(stream, offs, i);
            let mut side = Vec::new();
            // `materialize` reads the extent of line i from offsets[i..i+2]: hand it the stripped extent
            let r = materialize_ext(&ctx, &out, stream, lo as i32, hi as i32, i, &mut side);
            f(i, &stream[lo..hi], r, &side);
        }
        true
    }

    /// Framing + UTF-8 validation + decode + `GelfEncoder::encode` of a raw stream on the device
    /// (`fg_split_decode_encode_gelf`, input.format = "rfc5424", "rfc3164", "ltsv" or "gelf", see `fuses_with_gelf`):
    /// `f(line, Ok(json) | Err(error), side)` in stream order, `line` without its terminator, `side` the decoder's
    /// println! lines for it (LTSV's "Missing value" lines, from `fg_encoded_ltsv_stops`); `json` carries the frame of
    /// `out_framing` (output.framing, `fg_set_output_framing`).  Then `all(bytes)` with the framed records of the whole
    /// call, the bytes one Output writes for them.  false (nothing decoded) when the stream does not fit the context.
    pub fn split_decode_encode_gelf<F: FnMut(&[u8], Result<&[u8], &'static str>, &[String]), G: FnOnce(&[u8])>(
        &self, stream: &[u8], extra: &[(String, String)], out_framing: fg_out_framing, f: F, all: G) -> bool {
        self.split_decode_encode(FusedOutput::Gelf, stream, extra, &[], out_framing, f, all)
    }

    /// `split_decode_encode_gelf` for any fused encoder: `output` = output.format, `extra` = its extras
    /// (output.gelf_extra, output.ltsv_extra or output.capnp_extra); with `FusedOutput::Ltsv` the records are
    /// `LTSVEncoder::encode`'s text (`fg_split_decode_encode_ltsv`), with `FusedOutput::Capnp` `CapnpEncoder::encode`'s
    /// messages (`fg_split_decode_encode_capnp`), with `FusedOutput::Passthrough` `prefix` + Record.full_msg
    /// (`fg_split_decode_encode_passthrough`; `prefix` is the header of this call, `extra` is not used).
    pub fn split_decode_encode<F: FnMut(&[u8], Result<&[u8], &'static str>, &[String]), G: FnOnce(&[u8])>(
        &self, output: FusedOutput, stream: &[u8], extra: &[(String, String)], prefix: &[u8], out_framing: fg_out_framing, mut f: F,
        all: G) -> bool {
        let mut ctx = self.ctx.lock().unwrap();
        assert_eq!(unsafe { fg_set_output_framing(ctx.raw, out_framing) }, 0);
        let o = output as usize;
        if output == FusedOutput::Passthrough {  // set on every call: the header carries the time of the call
            assert_eq!(unsafe { fg_set_passthrough_prefix(ctx.raw, prefix.as_ptr(), prefix.len() as i64) }, 0);
        } else if ctx.extra[o].as_deref() != Some(extra) {
            let keys: Vec<CString> = extra.iter().map(|(k, _)| CString::new(k.as_str()).unwrap()).collect();
            let vals: Vec<CString> = extra.iter().map(|(_, v)| CString::new(v.as_str()).unwrap()).collect();
            let kp: Vec<*const c_char> = keys.iter().map(|s| s.as_ptr()).collect();
            let vp: Vec<*const c_char> = vals.iter().map(|s| s.as_ptr()).collect();
            let set = match output {
                FusedOutput::Gelf => fg_set_gelf_extra,
                FusedOutput::Ltsv => fg_set_ltsv_extra,
                FusedOutput::Capnp => fg_set_capnp_extra,
                FusedOutput::Passthrough => unreachable!(),
            };
            assert_eq!(unsafe { set(ctx.raw, kp.len() as i32, kp.as_ptr(), vp.as_ptr()) }, 0);
            ctx.extra[o] = Some(extra.to_vec());
        }
        let mut out: fg_encoded_out = unsafe { std::mem::zeroed() };
        let mut lines: *const i32 = ptr::null();
        let call = match output {
            FusedOutput::Gelf => fg_split_decode_encode_gelf,
            FusedOutput::Ltsv => fg_split_decode_encode_ltsv,
            FusedOutput::Capnp => fg_split_decode_encode_capnp,
            FusedOutput::Passthrough => fg_split_decode_encode_passthrough,
        };
        let rc = unsafe { call(ctx.raw, ctx.fmt, fg_framing_FG_FRAME_LINE, stream.as_ptr(), stream.len() as i64, &mut out, &mut lines) };
        if rc == FG_E_CAPACITY {
            return false;
        }
        if rc != 0 {
            let e = unsafe { CStr::from_ptr(fg_last_error(ctx.raw)) }.to_string_lossy().into_owned();
            panic!("fused decode + encode: {}", e);
        }
        let n = out.n as usize;
        let offs = unsafe { std::slice::from_raw_parts(lines, n + 1) };
        let mut stops: *const i32 = ptr::null();
        if ctx.fmt == fg_format_FG_FMT_LTSV {
            assert_eq!(unsafe { fg_encoded_ltsv_stops(ctx.raw, &mut stops) }, 0);
        }
        let mut side = Vec::new();
        for i in 0..n {
            let (lo, hi) = line_extent(stream, offs, i);
            side.clear();
            let stop = if stops.is_null() { -1 } else { unsafe { *stops.add(i) } };
            if stop >= 0 {
                // a record with a stop passed the UTF-8 check
                missing_values(unsafe { std::str::from_utf8_unchecked(&stream[lo..hi]) }, stop as usize, &mut side);
            }
            let (st, a, b) = unsafe { (*out.status.add(i), *out.offsets.add(i) as usize, *out.offsets.add(i + 1) as usize) };
            if st == 0 {
                f(&stream[lo..hi], Ok(unsafe { std::slice::from_raw_parts(out.bytes.add(a), b - a) }), &side);
            } else {
                f(&stream[lo..hi], Err(error_str(ctx.fmt, st as u32)), &side);
            }
        }
        all(unsafe { std::slice::from_raw_parts(out.bytes, *out.offsets.add(n) as usize) });
        true
    }
}

/// The lines of `block` in stream order through `run`, which returns false when they do not fit the context it is given:
/// such a block is decoded in two halves cut after a '\n' near its middle, and a lone line longer than the context's
/// max_batch_bytes on a context of its own, sized for it (rare, slow, correct: the reference takes lines of any length).
fn decode_fitting<F: FnMut(&CudaDecoder, &[u8]) -> bool>(gpu: &CudaDecoder, block: &[u8], run: &mut F) {
    let n = block.len();
    if n == 0 || (n <= gpu.capacity_bytes() && run(gpu, block)) {
        return;
    }
    let mid = n / 2;
    // the last byte ends the last line: it is no cut
    let cut = block[mid..n - 1].iter().position(|&c| c == b'\n').map(|p| mid + p + 1)
        .or_else(|| block[..mid].iter().rposition(|&c| c == b'\n').map(|p| p + 1));
    match cut {
        Some(c) => {
            decode_fitting(gpu, &block[..c], run);
            decode_fitting(gpu, &block[c..], run);
        }
        None => {
            let big = gpu.make_sized(n + 4096);
            assert!(run(&big, block), "a line does not fit a context sized for it");
        }
    }
}

/// Reads RAW BLOCKS of `max_bytes` or more (no per-line `String`), cuts each block after its last '\n' and hands the
/// whole lines to `flush`, keeping the unterminated tail for the next block; at EOF the rest, an unterminated last line
/// included.
fn run_blocks<T: Read, F: FnMut(&[u8])>(mut buf_reader: BufReader<T>, max_bytes: usize, mut flush: F) {
    let mut block: Vec<u8> = Vec::with_capacity(max_bytes);
    loop {
        let got = match buf_reader.fill_buf() {
            Ok(b) => { let n = b.len(); block.extend_from_slice(b); n }
            Err(e) => match e.kind() {
                ErrorKind::Interrupted => continue,
                ErrorKind::WouldBlock => {
                    flush(&block);
                    let _ = writeln!(stderr(), "Client hasn't sent any data for a while - Closing idle connection");
                    return;
                }
                _ => { flush(&block); return; }
            },
        };
        buf_reader.consume(got);
        if got == 0 {                       // EOF: an unterminated last line is still a line
            flush(&block);
            return;
        }
        if block.len() >= max_bytes {
            // decode every complete line of the block, keep the unterminated tail for the next one
            let cut = block.iter().rposition(|&c| c == b'\n').map_or(0, |p| p + 1);
            if cut > 0 {
                flush(&block[..cut]);
                block.drain(..cut);
            }
        }
    }
}

fn span<'a>(bytes: &'a [u8], s: fg_span) -> &'a str {
    // spans delimit whole UTF-8 sequences of a line that was validated before the call
    unsafe { std::str::from_utf8_unchecked(&bytes[s.off as usize..(s.off + s.len) as usize]) }
}

/// JSON string body already validated on the device -> String; `nl_retry` = gelf_decoder.rs:44-46 semantics.
fn json_unescape(v: &str, nl_retry: bool) -> String {
    let b = v.as_bytes();
    let mut out = String::with_capacity(b.len());
    let hex = |s: &[u8]| s.iter().fold(0u32, |n, &c| n * 16 + (c as char).to_digit(16).unwrap());
    let mut i = 0;
    let mut raw_from = 0;
    while i < b.len() {
        if b[i] != b'\\' { i += 1; continue; }
        out.push_str(&v[raw_from..i]);
        let e = b[i + 1];
        i += 2;
        match e {
            b'"' => out.push('"'), b'\\' => out.push('\\'), b'/' => out.push('/'),
            b'b' => out.push('\x08'), b'f' => out.push('\x0c'), b'n' => out.push('\n'),
            b'r' => out.push('\r'), b't' => out.push('\t'),
            b'u' => {
                let mut n = hex(&b[i..i + 4]);
                i += 4;
                if (0xD800..=0xDBFF).contains(&n) {
                    let n2 = hex(&b[i + 2..i + 6]);
                    i += 6;
                    n = (((n - 0xD800) << 10) | (n2 - 0xDC00)) + 0x1_0000;
                }
                out.push(std::char::from_u32(n).unwrap());
            }
            b'\n' if nl_retry => out.push_str("\\n"),
            _ => {}
        }
        raw_from = i;
    }
    out.push_str(&v[raw_from..]);
    out
}

fn materialize(ctx: &Ctx, out: &fg_batch_out, bytes: &[u8], offsets: &[i32], i: usize, side: &mut Vec<String>) -> Result<Record, &'static str> {
    materialize_ext(ctx, out, bytes, offsets[i], offsets[i + 1], i, side)
}

/// RFC5424: compact 32-byte row (`fg_row5424`) + 8-byte entries; escaped SD values were unescaped ON THE DEVICE
/// (rfc5424_decoder.rs:105-125) and live in `out.arena`.  Rows flagged FG_FLAG_WIDE carry absolute spans instead.
unsafe fn materialize_5424(ctx: &Ctx, out: &fg_batch_out, bytes: &[u8], line_lo: i32, i: usize) -> Result<Record, &'static str> {
    let row = &*out.rows5424.add(i);
    let status = row.meta & 0xFF;
    if status != 0 {
        let s = CStr::from_ptr(fg_error_string(ctx.fmt, status));
        return Err(std::str::from_utf8_unchecked(std::slice::from_raw_parts(s.as_ptr() as *const u8, s.to_bytes().len())));
    }
    let (fac, sev, flags) = ((row.meta >> 8) & 0xFF, (row.meta >> 16) & 0xFF, row.meta >> 24);
    let arena = |off: u32, len: usize| std::str::from_utf8_unchecked(std::slice::from_raw_parts(out.arena.add(off as usize), len)).to_owned();
    if flags & FG_FLAG_WIDE != 0 {
        let w = &*out.wide_rows.add(row.sd_first as usize);
        let mut sd: Vec<StructuredData> = Vec::new();
        for e in w.sd.off..w.sd.off + w.sd.len {
            let e = e as usize;
            let em = *out.entry_meta.add(e) as u32;
            let nm = *out.entry_name.add(e);
            if em & FG_EM_TAG_MASK == fg_tag_FG_TAG_SD_HEADER as u32 {
                sd.push(StructuredData::new(Some(span(bytes, nm))));
                continue;
            }
            let val = *out.entry_val.add(e);
            let v = if em & FG_EM_ARENA != 0 { arena(val as u32, (val >> 32) as usize) }
                    else { span(bytes, fg_span { off: (val & 0xFFFF_FFFF) as i32, len: (val >> 32) as i32 }).to_owned() };
            sd.last_mut().unwrap().pairs.push((format!("_{}", span(bytes, nm)), SDValue::String(v)));
        }
        return Ok(Record {
            ts: w.ts, hostname: span(bytes, w.hostname).to_owned(), facility: Some(fac as u8), severity: Some(sev as u8),
            appname: Some(span(bytes, w.appname).to_owned()), procid: Some(span(bytes, w.procid).to_owned()),
            msgid: Some(span(bytes, w.msgid).to_owned()),
            msg: if w.msg.off >= 0 { Some(span(bytes, w.msg).to_owned()) } else { None },
            full_msg: Some(span(bytes, w.full_msg).to_owned()),
            sd: if sd.is_empty() { None } else { Some(sd) },
        });
    }
    let line = &bytes[line_lo as usize..];
    let rel = |a: usize, b: usize| std::str::from_utf8_unchecked(&line[a..b]).to_owned();
    let sp: Vec<usize> = row.sp.iter().map(|&x| x as usize).collect();
    let (mo, ml) = (row.msg_off as usize, row.msg_len as usize);
    let mut sd: Vec<StructuredData> = Vec::new();
    let mut e = row.sd_first as usize;
    let end = e + row.sd_count as usize;
    while e < end {
        let v = *out.entries8.add(e);
        let (a, b, c) = ((v & 0xFFFF) as usize, ((v >> 16) & 0xFFFF) as usize, ((v >> 32) & 0xFFFF) as usize);
        if v & FG_E8_HEADER != 0 {
            sd.push(StructuredData::new(Some(&rel(a, b))));
        } else {
            let value = if v & FG_E8_ARENA != 0 {
                let off = (((v >> 32) & 0x3FFF_FFFF) as u32) << 1;   // record = [u16 length][bytes]
                let len = u16::from_le_bytes([*out.arena.add(off as usize), *out.arena.add(off as usize + 1)]) as usize;
                arena(off + 2, len)
            } else {
                rel(b + 2, c)
            };
            sd.last_mut().unwrap().pairs.push((format!("_{}", rel(a, b)), SDValue::String(value)));   // :221
        }
        e += 1;
    }
    Ok(Record {
        ts: row.ts, hostname: rel(sp[0] + 1, sp[1]), facility: Some(fac as u8), severity: Some(sev as u8),
        appname: Some(rel(sp[1] + 1, sp[2])), procid: Some(rel(sp[2] + 1, sp[3])), msgid: Some(rel(sp[3] + 1, sp[4])),
        msg: if ml > 0 { Some(rel(mo, mo + ml)) } else { None },
        full_msg: Some(rel(0, mo + ml)),
        sd: if sd.is_empty() { None } else { Some(sd) },
    })
}

/// The println! of ltsv_decoder.rs:99: "Missing value for name '{part}'" for every tab-separated part of `line` without
/// ':' that starts before `stop` (relative to the line; `line.len() + 1` = every part)
fn missing_values(line: &str, stop: usize, side: &mut Vec<String>) {
    let mut a = 0;
    for part in line.split('\t') {
        if a >= stop { break; }
        if !part.contains(':') { side.push(format!("Missing value for name '{}'", part)); }
        a += part.len() + 1;
    }
}

fn materialize_ext(ctx: &Ctx, out: &fg_batch_out, bytes: &[u8], line_lo: i32, line_hi: i32, i: usize, side: &mut Vec<String>) -> Result<Record, &'static str> {
    unsafe {
        if !out.rows5424.is_null() {
            return materialize_5424(ctx, out, bytes, line_lo, i);
        }
        let meta = *out.meta.add(i);
        let status = meta & 0xFF;
        let flags = (meta >> 24) & 0xFF;
        if flags & FG_FLAG_MISSING_VALUE != 0 {
            // all parts when Ok / post-loop error, else the parts before the failing one
            let (lo, hi) = (line_lo as usize, line_hi as usize);
            let stop = if status != 0 { (*out.full_msg.add(i)).off as usize } else { hi + 1 };
            missing_values(span(bytes, fg_span { off: lo as i32, len: (hi - lo) as i32 }), stop - lo, side);
        }
        if status != 0 {
            let s = CStr::from_ptr(fg_error_string(ctx.fmt, status));
            return Err(std::str::from_utf8_unchecked(std::slice::from_raw_parts(s.as_ptr() as *const u8, s.to_bytes().len())));
        }
        let nl = flags & FG_FLAG_NL_RETRY != 0;
        let opt = |col: *const fg_span| if col.is_null() || (*col.add(i)).off < 0 { None } else { Some(span(bytes, *col.add(i)).to_owned()) };
        let esc = |s: Option<String>, bit: u32| s.map(|x| if flags & bit != 0 { json_unescape(&x, nl) } else { x });
        let fac = (meta >> 8) & 0xFF;
        let sev = (meta >> 16) & 0xFF;
        let sd_span = *out.sd.add(i);
        let mut sd: Vec<StructuredData> = Vec::new();
        if sd_span.len > 0 {
            sd.push(StructuredData::new(None));  // LTSV / GELF: one element without sd_id
            for e in sd_span.off..sd_span.off + sd_span.len {
                let e = e as usize;
                let em = *out.entry_meta.add(e) as u32;
                let tag = em & FG_EM_TAG_MASK;
                let nm = *out.entry_name.add(e);
                if tag == fg_tag_FG_TAG_SD_HEADER as u32 {
                    sd.push(StructuredData::new(if nm.off >= 0 { Some(span(bytes, nm)) } else { None }));
                    continue;
                }
                let mut name = String::new();
                if em & FG_EM_NO_PREFIX == 0 { name.push('_'); }
                if em & FG_EM_NAME_ESC != 0 { name.push_str(&json_unescape(span(bytes, nm), nl)); } else { name.push_str(span(bytes, nm)); }
                if em & FG_EM_SUFFIX != 0 { if let Some(ref s) = ctx.suffix[tag as usize] { name.push_str(s); } }
                let val = *out.entry_val.add(e);
                let v = match tag {
                    0 => {
                        let raw = span(bytes, fg_span { off: (val & 0xFFFF_FFFF) as i32, len: (val >> 32) as i32 });
                        SDValue::String(if em & FG_EM_UNESCAPE == 0 { raw.to_owned() } else { json_unescape(raw, nl) })
                    }
                    1 => SDValue::Bool(val != 0),
                    2 => SDValue::F64(f64::from_bits(val)),
                    3 => SDValue::I64(val as i64),
                    4 => SDValue::U64(val),
                    _ => SDValue::Null,
                };
                sd.last_mut().unwrap().pairs.push((name, v));
            }
        }
        let ts = if flags & FG_FLAG_TS_MISSING != 0 {
            flowgger::flowgger::utils::PreciseTimestamp::now().as_f64() // gelf_decoder.rs:109
        } else {
            *out.ts.add(i)
        };
        Ok(Record {
            ts,
            hostname: esc(opt(out.hostname), FG_FLAG_HOST_ESC).unwrap_or_default(),
            facility: if fac != 0xFF { Some(fac as u8) } else { None },
            severity: if sev != 0xFF { Some(sev as u8) } else { None },
            appname: opt(out.appname),
            procid: opt(out.procid),
            msgid: opt(out.msgid),
            msg: if flags & FG_FLAG_MSG_ARENA != 0 {
                // RFC3164: the message tokens re-joined by single spaces on the device (rfc3164_decoder.rs:67)
                let m = *out.msg.add(i);
                Some(std::str::from_utf8_unchecked(std::slice::from_raw_parts(out.arena.add(m.off as usize), m.len as usize)).to_owned())
            } else {
                esc(opt(out.msg), FG_FLAG_MSG_ESC)
            },
            full_msg: esc(opt(out.full_msg), FG_FLAG_FULL_ESC),
            sd: if sd.is_empty() { None } else { Some(sd) },
        })
    }
}

impl Decoder for CudaDecoder {
    /// Drop-in single-line form: a batch of one through the same kernels.
    fn decode(&self, line: &str) -> Result<Record, &'static str> {
        let offsets = [0i32, line.len() as i32];
        let mut res = Err("unreachable");
        self.decode_batch(line.as_bytes(), &offsets, |_, r, side| {
            for s in side { println!("{}", s); }
            res = r;
        });
        res
    }
}

/// Batched twin of `LineSplitter` (src/flowgger/splitter/line_splitter.rs:10-54): inserted between `input` and
/// `decoder`.  It reads RAW BLOCKS (no per-line `String`), cuts each block after its last '\n' and hands the block to
/// `fg_split_decode`: line framing (`BufRead::lines`: "\n", one "\r"), the UTF-8 check of `String` and the decode all run
/// on the device; stderr text and record order are those of the reference.  A block that holds more lines than the
/// context is decoded in halves, and a line longer than the context's max_batch_bytes on a context sized for it.
pub struct BatchingLineSplitter {
    pub gpu: CudaDecoder,
    pub max_bytes: usize,
}

impl BatchingLineSplitter {
    fn flush<F: FnMut(Vec<u8>)>(&self, block: &[u8], encoder: &Box<dyn Encoder>, send: &mut F) {
        decode_fitting(&self.gpu, block, &mut |gpu: &CudaDecoder, part: &[u8]| {
            gpu.split_decode(part, |_, line, r, side| {
                for s in side { println!("{}", s); }
                match r.and_then(|rec| encoder.encode(rec)) {
                    Ok(bytes) => send(bytes),
                    Err("Invalid UTF-8 input") => { let _ = writeln!(stderr(), "Invalid UTF-8 input"); }   // line_splitter.rs:22-25
                    Err(e) => { let _ = writeln!(stderr(), "{}: [{}]", e, String::from_utf8_lossy(line).trim()); }  // :37-39
                }
            })
        });
    }
}

impl<T: Read> Splitter<T> for BatchingLineSplitter {
    fn run(&self, buf_reader: BufReader<T>, tx: SyncSender<Vec<u8>>, _decoder: Box<dyn Decoder>, encoder: Box<dyn Encoder>) {
        let mut send = |bytes: Vec<u8>| tx.send(bytes).unwrap();
        let max_bytes = self.max_bytes.min(self.gpu.capacity_bytes());
        run_blocks(buf_reader, max_bytes, |block| self.flush(block, &encoder, &mut send));
    }
}

/// The `input.format` values whose decoder runs fused with the GELF encoder on the device (`fg_decode_encode_gelf`,
/// `fg_split_decode_encode_gelf`); `FusedGelfLineSplitter` takes a `CudaDecoder` of one of them.
pub fn fuses_with_gelf(input_format: &str) -> bool {
    matches!(input_format, "rfc5424" | "rfc3164" | "ltsv" | "gelf")
}

/// The `input.format` values whose decoder runs fused with the LTSV encoder on the device (`fg_decode_encode_ltsv`,
/// `fg_split_decode_encode_ltsv`): the same four; `FusedLtsvLineSplitter` takes a `CudaDecoder` of one of them.
pub fn fuses_with_ltsv(input_format: &str) -> bool {
    fuses_with_gelf(input_format)
}

/// The `input.format` values whose decoder runs fused with the Cap'n Proto encoder on the device
/// (`fg_decode_encode_capnp`, `fg_split_decode_encode_capnp`): the same four; `FusedCapnpLineSplitter` takes a
/// `CudaDecoder` of one of them.
pub fn fuses_with_capnp(input_format: &str) -> bool {
    fuses_with_gelf(input_format)
}

/// The `input.format` values whose decoder runs fused with the passthrough encoder on the device
/// (`fg_decode_encode_passthrough`, `fg_split_decode_encode_passthrough`): the same four;
/// `FusedPassthroughLineSplitter` takes a `CudaDecoder` of one of them.
pub fn fuses_with_passthrough(input_format: &str) -> bool {
    fuses_with_gelf(input_format)
}

/// The output format of a fused encoder (output.format = "gelf", "ltsv", "capnp" or "passthrough")
#[derive(Clone, Copy, PartialEq, Eq, Debug)]
pub enum FusedOutput {
    Gelf = 0,
    Ltsv = 1,
    Capnp = 2,
    Passthrough = 3,
}

/// The device framing of an `output.framing` value, as `mod.rs:453-460` picks the merger (panics on an unknown one, as
/// the reference does)
pub fn out_framing_of(output_framing: &str) -> fg_out_framing {
    match output_framing {
        "noop" | "nop" | "none" | "capnp" => fg_out_framing_FG_OUT_NONE,
        "line" => fg_out_framing_FG_OUT_LINE,
        "nul" => fg_out_framing_FG_OUT_NUL,
        "syslen" => fg_out_framing_FG_OUT_SYSLEN,
        _ => panic!("Invalid framing type: {}", output_framing),
    }
}

/// `output.format = "gelf"` with `input.format = "rfc5424"`, `"rfc3164"`, `"ltsv"` or `"gelf"` (`fuses_with_gelf`): framing, the
/// UTF-8 check, decode AND encode run on the device (`fg_split_decode_encode_gelf`, replaces BufRead::lines +
/// Decoder::decode + GelfEncoder::encode of line_splitter.rs:17-52); it reads raw blocks like `BatchingLineSplitter` and
/// only the encoded records come back.  An RFC3164 context fixes the year of year-less timestamps at the start of each
/// call; an LTSV context's "Missing value" lines are printed to stdout before their record is sent or reported.  A GELF
/// context (a GELF relay) stamps every record without "timestamp" with the wall clock read once at the start of each call
/// (`fg_encoded_gelf_now`) rather than per record, and re-escapes strings from their unescaped text.
/// With `out_framing` other than `FG_OUT_NONE` the device also applies output.framing (merger/*.rs) and the splitter
/// sends ONE `Vec` per block, the framed records of the whole block: the Output must then be started without a merger.
pub struct FusedGelfLineSplitter {
    pub gpu: CudaDecoder,
    pub extra: Vec<(String, String)>,   // output.gelf_extra (gelf_encoder.rs:29-48)
    pub out_framing: fg_out_framing,    // output.framing (mod.rs:444-460), resolved by the caller
    pub max_bytes: usize,
}

impl<T: Read> Splitter<T> for FusedGelfLineSplitter {
    fn run(&self, buf_reader: BufReader<T>, tx: SyncSender<Vec<u8>>, _decoder: Box<dyn Decoder>, _encoder: Box<dyn Encoder>) {
        run_fused(&self.gpu, FusedOutput::Gelf, &self.extra, None, self.out_framing, self.max_bytes, buf_reader, tx)
    }
}

/// `output.format = "ltsv"` with `input.format` one of `fuses_with_ltsv`: `FusedGelfLineSplitter` with the LTSV encoder
/// (`fg_split_decode_encode_ltsv`, replaces Decoder::decode + LTSVEncoder::encode, ltsv_encoder.rs:66-123).  The caller
/// resolves output.framing's default, "line" for ltsv (mod.rs:444-460).
pub struct FusedLtsvLineSplitter {
    pub gpu: CudaDecoder,
    pub extra: Vec<(String, String)>,   // output.ltsv_extra (ltsv_encoder.rs:10-30), in byte order of the keys
    pub out_framing: fg_out_framing,    // output.framing (mod.rs:444-460), resolved by the caller
    pub max_bytes: usize,
}

impl<T: Read> Splitter<T> for FusedLtsvLineSplitter {
    fn run(&self, buf_reader: BufReader<T>, tx: SyncSender<Vec<u8>>, _decoder: Box<dyn Decoder>, _encoder: Box<dyn Encoder>) {
        run_fused(&self.gpu, FusedOutput::Ltsv, &self.extra, None, self.out_framing, self.max_bytes, buf_reader, tx)
    }
}

/// `output.format = "capnp"` with `input.format` one of `fuses_with_capnp`: `FusedGelfLineSplitter` with the Cap'n Proto
/// encoder (`fg_split_decode_encode_capnp`, replaces Decoder::decode + CapnpEncoder::encode, capnp_encoder.rs:36-109).
/// The caller resolves output.framing's default, "noop" for capnp (mod.rs:444-460): `FG_OUT_NONE`, one `Vec` per record.
pub struct FusedCapnpLineSplitter {
    pub gpu: CudaDecoder,
    pub extra: Vec<(String, String)>,   // output.capnp_extra (capnp_encoder.rs:14-32), in byte order of the keys
    pub out_framing: fg_out_framing,    // output.framing (mod.rs:444-460), resolved by the caller
    pub max_bytes: usize,
}

impl<T: Read> Splitter<T> for FusedCapnpLineSplitter {
    fn run(&self, buf_reader: BufReader<T>, tx: SyncSender<Vec<u8>>, _decoder: Box<dyn Decoder>, _encoder: Box<dyn Encoder>) {
        run_fused(&self.gpu, FusedOutput::Capnp, &self.extra, None, self.out_framing, self.max_bytes, buf_reader, tx)
    }
}

/// `output.format = "passthrough"` with `input.format` one of `fuses_with_passthrough`: `FusedGelfLineSplitter` with the
/// passthrough encoder (`fg_split_decode_encode_passthrough`, replaces Decoder::decode + PassthroughEncoder::encode,
/// passthrough_encoder.rs:22-46): each record is the header + Record.full_msg, and a GELF record without full_message
/// prints "Cannot output empty raw message: [line]" on stderr.  The header (output.syslog_prepend_timestamp) is
/// formatted once per device call, as build_prepend_ts does per record (encoder/mod.rs:82-94), so it can differ from
/// the reference's for the records encoded after the clock crossed a tick of the format's finest field during the call.
/// The caller resolves output.framing's default (mod.rs:444-451): "noop", `FG_OUT_NONE`, or "line" for output.type =
/// "debug".
pub struct FusedPassthroughLineSplitter {
    pub gpu: CudaDecoder,
    pub header_format: Option<String>,  // config_get_prepend_ts (encoder/mod.rs:58-80): validated, None without a header
    pub out_framing: fg_out_framing,    // output.framing (mod.rs:444-451), resolved by the caller
    pub max_bytes: usize,
}

impl FusedPassthroughLineSplitter {
    /// None when output.syslog_prepend_timestamp is not a format description build_prepend_ts can use: the reference
    /// then fails every record that has a full_msg ("Failed to format date when building prepend timestamp for header
    /// while encoding Passthrough"), which the caller keeps by running LineSplitter with PassthroughEncoder instead.
    pub fn new(gpu: CudaDecoder, config: &Config, out_framing: fg_out_framing, max_bytes: usize) -> Option<FusedPassthroughLineSplitter> {
        let header_format = config_get_prepend_ts(config);
        if let Some(f) = &header_format {
            build_prepend_ts(f).ok()?;
        }
        Some(FusedPassthroughLineSplitter { gpu, header_format, out_framing, max_bytes })
    }
}

impl<T: Read> Splitter<T> for FusedPassthroughLineSplitter {
    fn run(&self, buf_reader: BufReader<T>, tx: SyncSender<Vec<u8>>, _decoder: Box<dyn Decoder>, _encoder: Box<dyn Encoder>) {
        run_fused(&self.gpu, FusedOutput::Passthrough, &[], self.header_format.as_deref(), self.out_framing, self.max_bytes, buf_reader, tx)
    }
}

fn run_fused<T: Read>(gpu: &CudaDecoder, output: FusedOutput, extra: &[(String, String)], header_format: Option<&str>,
                      out_framing: fg_out_framing, max_bytes: usize, buf_reader: BufReader<T>, tx: SyncSender<Vec<u8>>) {
    let max_bytes = max_bytes.min(gpu.capacity_bytes());
    let framed = out_framing != fg_out_framing_FG_OUT_NONE;
    run_blocks(buf_reader, max_bytes, |block| {
        decode_fitting(gpu, block, &mut |gpu: &CudaDecoder, part: &[u8]| {
            // the passthrough header of this device call (FusedPassthroughLineSplitter::new checked that it formats)
            let prefix = header_format.map_or(String::new(), |f| build_prepend_ts(f).expect("syslog_prepend_timestamp"));
            gpu.split_decode_encode(output, part, extra, prefix.as_bytes(), out_framing, |line, r, side| {
                for s in side { println!("{}", s); }  // ltsv_decoder.rs:99
                match r {
                    Ok(rec) => if !framed { tx.send(rec.to_vec()).unwrap() },
                    Err("Invalid UTF-8 input") => { let _ = writeln!(stderr(), "Invalid UTF-8 input"); }   // line_splitter.rs:22-25
                    Err(e) => { let _ = writeln!(stderr(), "{}: [{}]", e, String::from_utf8_lossy(line).trim()); }  // :37-39
                }
            }, |all| if framed && !all.is_empty() { tx.send(all.to_vec()).unwrap() })
        })
    });
}

"""Framing on the device vs on the host for the fused GELF pipelines (output.format = "gelf", input.format = "rfc5424",
the default pair, "rfc3164", "ltsv" or "gelf").

    python tools/bench_split_encode.py [--format rfc5424|rfc3164|ltsv|gelf] [--ltsv-typed] [--lines 10000000] [--steps 10]
                                       [--warmup 2] [--splitter-gb 1.0] [--splitter-only] [--out-framing none|line|nul|syslen]

On the workload of bench.py for the format (rfc5424: C2, seed 5424; rfc3164: seed 3164, year 2026; ltsv: seed 1757,
with --ltsv-typed bench.py's schema and suffixes; gelf: bench.py's seed; the same mean line length), joined with '\\n' in pinned memory:
  1. fg_split_decode_encode_gelf on the raw stream and fg_decode_encode_gelf on the same lines framed beforehand (for
     rfc3164, ltsv and gelf also fg_split_decode on the raw stream: decode only, rows + side tables back), timed alternately
     after warm-ups; the two encoding calls must return byte-identical records, statuses and (ltsv) "Missing value" stops
     (gelf: a record without "timestamp" carries its call's wall clock, which is swapped for the other call's first);
  2. the C++ BatchingLineSplitter with the fused GELF encoder end to end over at least --splitter-gb of the same text
     (text in, every JSON record handed to the sender, stderr captured).
--out-framing applies output.framing on the device (fg_set_output_framing) in both sections: the encoding calls return the
framed output stream, and the splitter sends one buffer per device call.
Prints one JSON line per section, with the card's name and power limit.  --splitter-only runs section 2 alone."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))

import bench  # noqa: E402
import flowgger_b200 as fb  # noqa: E402

# bench.py: SEEDS, GEN_MEAN and RFC3164_YEAR (the year of a timestamp without one, fixed so that a run is reproducible)
WORKLOADS = {"rfc5424": (fb.FMT_RFC5424, 5424, 169.2), "rfc3164": (fb.FMT_RFC3164, 3164, 140.0),
             "ltsv": (fb.FMT_LTSV, bench.SEEDS["ltsv"], bench.GEN_MEAN["ltsv"]),
             "gelf": (fb.FMT_GELF, bench.SEEDS["gelf"], bench.GEN_MEAN["gelf"])}
RFC3164_YEAR = 2026
OUT_FRAMINGS = {"none": fb.OUT_NONE, "line": fb.OUT_LINE, "nul": fb.OUT_NUL, "syslen": fb.OUT_SYSLEN}


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu": None, "error": str(e)}


def workload(fmt_name: str, n: int) -> tuple[np.ndarray, np.ndarray]:
    """the raw stream (every line followed by '\\n') and its line offsets, terminators included"""
    fmt, seed, mean = WORKLOADS[fmt_name]
    return fb.generate(fmt, seed, n, mean_len=mean, bad_frac=0.005, nthreads=32, terminated=True)


def same_clock(res, sb, so, pb, po):
    """GELF: the records of lines without "timestamp" carry the wall clock of their call.  Returns both calls' records
    with the split call's clock text replaced by the pre-framed call's (one record shows each), as bytes + offsets."""
    missing = np.flatnonzero(((res.meta & 0xFF) == 0) & (((res.meta >> 24) & 0x01) != 0))
    sb, pb = bytes(sb), bytes(pb)
    if len(missing) == 0:
        return sb, so, pb, po
    i = int(missing[0])

    def clock(buf, offs):
        rec = buf[offs[i]:offs[i + 1]]
        a = rec.index(b',"timestamp":') + len(b',"timestamp":')
        return rec[a:rec.index(b",", a)]  # "version" always follows

    ts, tp = clock(sb, so), clock(pb, po)
    sb = sb.replace(b',"timestamp":' + ts + b",", b',"timestamp":' + tp + b",")
    grow = np.zeros(len(so), np.int64)
    grow[missing + 1] = len(tp) - len(ts)
    so = so + np.cumsum(grow)
    return np.frombuffer(sb, np.uint8), so, np.frombuffer(pb, np.uint8), po


def decoder(fmt_name: str, typed: bool = False, **kw) -> fb.BatchDecoder:
    fmt = WORKLOADS[fmt_name][0]
    if fmt == fb.FMT_LTSV and typed:
        kw.update(ltsv_schema=bench.LTSV_SCHEMA, ltsv_suffixes=bench.LTSV_SUFFIXES)
    return fb.BatchDecoder(fmt, rfc3164_year=RFC3164_YEAR if fmt == fb.FMT_RFC3164 else 0, **kw)


def device_paths(args, stream: np.ndarray, soffs: np.ndarray, info: dict) -> None:
    n = len(soffs) - 1
    keep = stream != ord("\n")  # the generator puts no '\n' inside a line
    lines = stream[keep]
    loffs = (soffs - np.arange(n + 1, dtype=np.int64)).astype(np.int32)
    del keep
    cap = dict(max_batch_bytes=len(stream) + (1 << 20), max_batch_lines=n + 64)
    split, pre = decoder(args.format, args.ltsv_typed, **cap), decoder(args.format, args.ltsv_typed, **cap)
    decode = decoder(args.format, args.ltsv_typed, **cap) if args.format != "rfc5424" else None
    try:
        split.set_output_framing(OUT_FRAMINGS[args.out_framing])
        pre.set_output_framing(OUT_FRAMINGS[args.out_framing])
        hs = split.host_alloc(len(stream))
        hs[:] = stream
        hl = pre.host_alloc(len(lines))
        hl[:] = lines
        ho = pre.host_alloc(loffs.nbytes, dtype=np.int32)
        ho[:] = loffs
        del lines
        hd = None
        if decode is not None:
            hd = decode.host_alloc(len(stream))
            hd[:] = stream
        for _ in range(args.warmup):
            split.split_decode_encode_gelf(hs, copy=False)
            pre.decode_encode_gelf(hl, ho, copy=False)
            if decode is not None:
                decode.split_decode(hd)
        t = {"split": [], "pre": [], "decode": []}
        k = {"split": [], "pre": [], "decode": []}
        framing_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            _, _, _, _, km = split.split_decode_encode_gelf(hs, copy=False)
            t["split"].append(time.perf_counter() - t0)
            k["split"].append(km)
            framing_ms.append(split.last_split_ms())
            t0 = time.perf_counter()
            _, _, _, km = pre.decode_encode_gelf(hl, ho, copy=False)
            t["pre"].append(time.perf_counter() - t0)
            k["pre"].append(km)
            if decode is not None:
                t0 = time.perf_counter()
                res = decode.split_decode(hd)
                t["decode"].append(time.perf_counter() - t0)
                k["decode"].append(res.kernel_ms)
        sb, so, ss, sl, _ = split.split_decode_encode_gelf(hs, copy=False)
        pb, po, ps, _ = pre.decode_encode_gelf(hl, ho, copy=False)
        assert len(ss) == n and np.array_equal(sl, soffs), "the device framed other lines than the generator made"
        if args.format == "gelf":
            sb, so, pb, po = same_clock(decode.split_decode(hd), sb, so, pb, po)
        assert np.array_equal(so, po) and np.array_equal(ss, ps) and np.array_equal(sb, pb), \
            "fg_split_decode_encode_gelf and fg_decode_encode_gelf disagree"
        if args.format == "ltsv":
            assert np.array_equal(split.ltsv_stops(), pre.ltsv_stops()), "the two calls disagree on the Missing value stops"
        out_bytes = int(so[-1])
        sections = [("split", "fg_split_decode_encode_gelf (pinned raw stream in)", len(stream)),
                    ("pre", "fg_decode_encode_gelf (pinned lines + int32 offsets in, framed beforehand)", int(loffs[-1]) + loffs.nbytes)]
        if decode is not None:
            sections.append(("decode", "fg_split_decode (pinned raw stream in, decode only: rows + side tables back, no JSON)", len(stream)))
        for key, api, in_bytes in sections:
            med = float(np.median(t[key]))
            rec = {"section": key, "api": api, "lines": n, "input_bytes": in_bytes, "json_bytes": out_bytes,
                   "records": int((ss == 0).sum()), "steps": args.steps, "call_ms_median": med * 1e3,
                   "call_ms_min": min(t[key]) * 1e3, "call_ms_max": max(t[key]) * 1e3,
                   "lines_per_s": n / med, "input_gb_per_s": in_bytes / med / 1e9, "output_gb_per_s": out_bytes / med / 1e9,
                   "kernel_ms_median": float(np.median(k[key])), **info}
            if key == "split":
                rec["framing_stage_ms_median"] = float(np.median(framing_ms))
            if key == "decode":
                for x in ("json_bytes", "output_gb_per_s"):
                    del rec[x]
            print(json.dumps(rec), flush=True)
    finally:
        split.close()
        pre.close()
        if decode is not None:
            decode.close()


def splitter(args, stream: np.ndarray, info: dict) -> None:
    # pieces of ~400 MB of whole lines: the records of one call come back as one Python bytes object, which ctypes
    # copies with an int length (< 2 GiB), and the JSON is about 2.6 times the text
    piece = 400_000_000
    cuts = [0]
    while cuts[-1] < len(stream):
        end = min(len(stream), cuts[-1] + piece)
        cuts.append(cuts[-1] + int(np.flatnonzero(stream[cuts[-1]:end] == ord("\n"))[-1]) + 1 if end < len(stream) else end)
    texts = [stream[a:b].tobytes() for a, b in zip(cuts[:-1], cuts[1:])]
    want = int(args.splitter_gb * 1e9)
    framing = OUT_FRAMINGS[args.out_framing]
    end = b"\0" if framing == fb.OUT_NUL else b"\n"  # one per record sent

    def run(text):
        if framing == fb.OUT_NONE:  # one record per send, the harness puts a "\n" after each
            return fb.splitter_run_gelf(dec, text, max_lines=1 << 19, max_bytes=64 << 20)
        return fb.splitter_run_gelf_framed(dec, text, framing, max_lines=1 << 19, max_bytes=64 << 20)[:2]

    dec = decoder(args.format, args.ltsv_typed, max_batch_bytes=64 << 20, max_batch_lines=1 << 20)
    wall, in_bytes, json_bytes, lines, n_rec, n_err = 0.0, 0, 0, 0, 0, 0
    try:
        small = texts[0][: 1 << 20]
        run(small[: small.rindex(b"\n") + 1])  # warm-up
        k = 0
        while in_bytes < want:
            text = texts[k % len(texts)]
            k += 1
            t0 = time.perf_counter()
            records, err = run(text)
            wall += time.perf_counter() - t0
            r, e, t = records.count(end), err.count(b"\n"), text.count(b"\n")
            sent = len(records) - (r if framing == fb.OUT_NONE else 0)
            assert r + e == t, (r, e, t)
            n_rec, n_err, lines = n_rec + r, n_err + e, lines + t
            in_bytes += len(text)
            json_bytes += sent
    finally:
        dec.close()
    print(json.dumps({"section": "splitter", "api": "BatchingLineSplitter + CudaGelfEncoder (fgh_splitter_run_gelf / "
                      "fgh_splitter_run_gelf_framed: text in, records + stderr out, 64 MiB batches; wall time summed over calls "
                      "of ~400 MB; json_bytes = the bytes sent, frames included)", "calls": k,
                      "lines": lines, "input_bytes": in_bytes, "json_bytes": json_bytes, "records": n_rec, "stderr_lines": n_err,
                      "wall_s": wall, "lines_per_s": lines / wall, "input_gb_per_s": in_bytes / wall / 1e9,
                      "output_gb_per_s": json_bytes / wall / 1e9, **info}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--format", choices=sorted(WORKLOADS), default="rfc5424")
    ap.add_argument("--lines", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--splitter-gb", type=float, default=1.0)
    ap.add_argument("--splitter-only", action="store_true")
    ap.add_argument("--ltsv-typed", action="store_true", help="ltsv: bench.py's schema and suffixes")
    ap.add_argument("--out-framing", choices=sorted(OUT_FRAMINGS), default="none", help="output.framing, applied on the device")
    args = ap.parse_args()
    info = card()
    info["out_framing"] = args.out_framing
    if args.format != "rfc5424":
        info["format"] = args.format
    if args.format == "ltsv":
        info["ltsv_typed"] = args.ltsv_typed
    stream, soffs = workload(args.format, args.lines)
    if not args.splitter_only:
        device_paths(args, stream, soffs, info)
    splitter(args, stream, info)


if __name__ == "__main__":
    main()

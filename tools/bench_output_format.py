"""GELF, LTSV, Cap'n Proto and passthrough output side by side on the device, per input format: output.format = "gelf"
(fg_decode_encode_gelf), "ltsv" (fg_decode_encode_ltsv), "capnp" (fg_decode_encode_capnp) and "passthrough"
(fg_decode_encode_passthrough, no header) over the same pre-framed lines in pinned memory, timed alternately in one
process.

    python tools/bench_output_format.py [--lines 4000000] [--steps 10] [--warmup 2] [--formats rfc5424,rfc3164,ltsv,gelf]

The workloads are tools/bench_split_encode.py's (bench.py's seeds and mean line lengths; ltsv with bench.py's schema and
suffixes).  One JSON line per (input format, output format): kernel ms per call (CUDA events around the parse + encode
kernels, fg_encoded_out.kernel_ms, median), end-to-end lines/s (host wall clock around the whole call: H2D, kernels,
D2H of the records, median), output bytes, and the card's name and power limit read in the same run."""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO / "tools"))

import bench_split_encode as B  # noqa: E402

fb = B.fb


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lines", type=int, default=4_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--formats", default="rfc5424,rfc3164,ltsv,gelf")
    args = ap.parse_args()
    info = B.card()
    for name in args.formats.split(","):
        fmt, seed, mean = B.WORKLOADS[name]
        lines, loffs = fb.generate(fmt, seed, args.lines, mean_len=mean, bad_frac=0.005, nthreads=32)
        dec = B.decoder(name, typed=name == "ltsv", max_batch_bytes=len(lines) + (1 << 20), max_batch_lines=args.lines + 1)
        data = dec.host_alloc(len(lines))
        data[:] = lines
        offs = dec.host_alloc(4 * len(loffs), np.int32)
        offs[:] = loffs
        calls = {"gelf": dec.decode_encode_gelf, "ltsv": dec.decode_encode_ltsv, "capnp": dec.decode_encode_capnp,
                 "passthrough": dec.decode_encode_passthrough}
        km = {k: [] for k in calls}
        wall = {k: [] for k in calls}
        nbytes = {}
        for step in range(args.warmup + args.steps):
            for out, call in calls.items():
                t0 = time.perf_counter()
                buf, eo, st, ms = call(data, offs, copy=False)
                dt = time.perf_counter() - t0
                nbytes[out] = int(eo[-1])
                if step >= args.warmup:
                    km[out].append(ms)
                    wall[out].append(dt)
        for out in calls:
            rec = {"input": name, "output": out, "lines": args.lines, "kernel_ms": round(statistics.median(km[out]), 3),
                   "lines_per_s": round(args.lines / statistics.median(wall[out])), "out_bytes": nbytes[out], **info}
            print(json.dumps(rec), flush=True)
        dec.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""The bench.py inference workload at another class count: same synthetic random weights (Detector default init under seed 1)
at C classes, same timed forward + fused decode/NMS, same in-run parity check against the CPU oracle.

  python tools/bench_classes.py --classes 150 [any bench.py option: --steps K --warmup W --side S --batch B --input u8|f32 ...]

Prints bench.py's JSON line with "classes" added to "config".  C may be up to 192 - anchors (two 96-column output tiles)."""
import argparse
import contextlib
import functools
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--classes", type=int, default=80)
    args, rest = ap.parse_known_args()
    bench.CLASSES = args.classes                       # read at call time by the weights, the plans, decode/NMS and the parity check
    # the per-stage algorithmic bytes bind their class count as a default argument: pass it explicitly
    bench.algorithmic_bytes_per_image = functools.partial(bench.algorithmic_bytes_per_image, C=args.classes)
    sys.argv = [sys.argv[0]] + rest
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        bench.main()
    for line in out.getvalue().splitlines():
        try:
            d = json.loads(line)
        except ValueError:
            print(line)
            continue
        d.setdefault("config", {})["classes"] = args.classes
        print(json.dumps(d), flush=True)


if __name__ == "__main__":
    main()

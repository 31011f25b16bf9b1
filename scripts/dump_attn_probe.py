#!/usr/bin/env python3
"""Dump what the decode kernel's self- and cross-attention phases compute at d = 1280 (20 heads, 64 rows, 132 CTAs), through the phase
probe of a build, so that two builds can be compared bit for bit.

  python scripts/dump_attn_probe.py --lib build_a/libwhisper_b200.so --out a.npz
  python scripts/dump_attn_probe.py --lib build_b/libwhisper_b200.so --out b.npz
  python scripts/dump_attn_probe.py --compare a.npz b.npz

The inputs are those of tests/test_decode_attention_stream_gpu.py: scattered self-KV cells (unattended cells NaN), key counts 1 .. 448;
cross K / V with 1500 real keys of 1536 and zero padding, as the encoder leaves it.
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import actq  # noqa: E402
from test_decode_attention_stream_gpu import N_AUDIO_CTX, cross_case, run_cross, run_self, self_case  # noqa: E402

FORMATS = {"f16": actq.F16, "q4_0": actq.Q4_0, "q4_1": actq.Q4_1, "q5_0": actq.Q5_0, "q5_1": actq.Q5_1, "q8_0": actq.Q8_0,
           "q3_k": actq.Q3_K, "q4_k": actq.Q4_K, "q5_k": actq.Q5_K}


def dump(lib_path, out):
    lib = C.CDLL(lib_path)
    lib.wb200_last_error.restype = C.c_char_p
    case = self_case(20, actq.ROWS)
    q, kw = cross_case(20, 0)
    res = {}
    for name, wt in FORMATS.items():
        res[f"self_{name}"] = run_self(lib, wt, case, 132, 0).view(np.uint8)
        res[f"cross_{name}"] = run_cross(lib, wt, 132, 0, actq.ROWS, q, kw, N_AUDIO_CTX).view(np.uint8)
    np.savez(out, **res)
    print(f"{out}: {len(res)} arrays from {lib_path}")


def compare(a, b):
    A, B = np.load(a), np.load(b)
    bad = [k for k in sorted(set(A.files) | set(B.files)) if k not in A.files or k not in B.files or not np.array_equal(A[k], B[k])]
    for k in sorted(A.files):
        print(f"{k}: {'DIFFERENT' if k in bad else 'equal'}")
    print("all equal" if not bad else f"{len(bad)} arrays differ")
    return 0 if not bad else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib", default=os.path.join(ROOT, "whisper.cpp_b200", "libwhisper_b200.so"))
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2, metavar="NPZ")
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("--out or --compare is needed")
    dump(args.lib, args.out)


if __name__ == "__main__":
    main()

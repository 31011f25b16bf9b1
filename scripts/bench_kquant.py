#!/usr/bin/env python3
"""K-quant decoding (Q4_K by default, --wtype q3_k): the persistent decode kernel (64 rows per pass) against the kernel-per-op chain (8 rows per pass), in one process.

Model: synth.cached_model("large-v3", Q4_K, seed=0, fast_pool=True), the model of `bench.py --config 3` (or the Q3_K one).
Arms (the decoder layout is fixed when a context is created, so the switch is set before each context):
  new   -- default (tile-major K-quant records, persistent kernel)
  chain -- WB200_MEGAKERNEL=0
  f16   -- WB200_KQUANT_AS_F16=1 (optional, --f16): the file expanded to F16 on the host, persistent kernel
Workloads:
  a -- 64 x 30 s chunks, greedy, no timestamps, one whisper_full_parallel(ctx, p, pcm, n, 64) call (the shape of the default bench line)
  b -- beam 5 on --minutes of audio through whisper_full (the shape of config 3)
Repeats alternate the arms (new, chain, new, chain, ...) so that the run-to-run spread is visible next to the difference.
Prints one JSON line per run and a summary line per (workload, arm); the card and its power limit come from nvidia-smi.

  python scripts/bench_kquant.py [--repeats 2] [--minutes 3] [--workloads ab] [--f16]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import load_pkg  # noqa: E402

ARMS = {"new": {}, "chain": {"WB200_MEGAKERNEL": "0"}, "f16": {"WB200_KQUANT_AS_F16": "1"}}
SWITCHES = ("WB200_MEGAKERNEL", "WB200_KQUANT_AS_F16")
LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_char_p, C.c_void_p)
QUIET = LOG_CB(lambda level, text, ud: None)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def counters(L):
    a = (C.c_double * 8)(); L.wb200_counters(a, 8)
    return [a[i] for i in range(8)]


def tokens(L, ctx):
    return [[L.whisper_full_get_token_id(ctx, s, j) for j in range(L.whisper_full_n_tokens(ctx, s))] for s in range(L.whisper_full_n_segments(ctx))]


def run(pkg, model, arm, workload, pcm, n_chunks):
    for k in SWITCHES:
        os.environ.pop(k, None)
    os.environ.update(ARMS[arm])
    eng = pkg.WhisperB200(model, gpu_device=0)
    for k in SWITCHES:
        os.environ.pop(k, None)
    L = eng.L
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    buf = pcm.ctypes.data_as(C.c_void_p)
    if workload == "a":
        p = L.whisper_full_default_params(0); p.greedy.best_of = 1; p.no_timestamps = True
    else:
        p = L.whisper_full_default_params(1); p.beam_search.beam_size = 5
    p.print_progress = False; p.temperature_inc = 0.0; p.n_threads = 4
    call = (lambda: L.whisper_full_parallel(eng.ctx, p, buf, len(pcm), n_chunks)) if workload == "a" else (lambda: L.whisper_full(eng.ctx, p, buf, len(pcm)))
    if workload == "a":                                          # the first call sizes the context pool and captures nothing worth timing
        assert call() == 0, L.wb200_last_error()
    c0 = counters(L)
    t0 = time.perf_counter()
    rc = call()
    dt = time.perf_counter() - t0
    c1 = counters(L)
    assert rc == 0, L.wb200_last_error()
    toks = tokens(L, eng.ctx)
    eng.close()
    passes = c1[0] - c0[0]
    return {"workload": workload, "arm": arm, "xRT": len(pcm) / 16000.0 / dt, "wall_s": dt, "decode_passes": passes,
            "rows_per_pass": (c1[1] - c0[1]) / max(1.0, passes), "decode_gpu_ms_per_pass": (c1[2] - c0[2]) / max(1.0, passes),
            "decoded_tokens": sum(len(t) for t in toks)}, toks


def agreement(a, b):
    """share of segments with identical token streams, and of tokens inside the common prefix of each segment pair"""
    same = sum(1 for x, y in zip(a, b) if x == y)
    pref = 0
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            if u != v:
                break
            pref += 1
    return {"segments": [len(a), len(b)], "identical_segments": same, "prefix_tokens": pref, "tokens": [sum(map(len, a)), sum(map(len, b))]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--minutes", type=float, default=3.0, help="audio of workload b")
    ap.add_argument("--workloads", default="ab")
    ap.add_argument("--f16", action="store_true", help="add the WB200_KQUANT_AS_F16=1 arm")
    ap.add_argument("--wtype", choices=("q4_k", "q3_k"), default="q4_k", help="block format of the synthetic large-v3 model")
    args = ap.parse_args()
    pkg = load_pkg(); synth = pkg.synth
    if not os.environ.get("WB200_VERBOSE"):                     # the library's INFO lines off stdout (whisper_log_set)
        lib = C.CDLL(pkg.LIB_PATH)
        lib.whisper_log_set.argtypes = [LOG_CB, C.c_void_p]
        lib.whisper_log_set(QUIET, None)
    model = synth.cached_model("large-v3", {"q4_k": synth.Q4_K, "q3_k": synth.Q3_K}[args.wtype], seed=0, fast_pool=True)
    arms = ["new", "chain"] + (["f16"] if args.f16 else [])
    gpu = card()
    inputs = {"a": (np.concatenate([synth.synth_audio(seed=i, seconds=30.0) for i in range(64)]), 64),
              "b": (np.concatenate([synth.synth_audio(seed=1234 + i, seconds=30.0) for i in range(max(1, int(round(args.minutes * 2))))]), 1)}
    summary = {}
    for w in args.workloads:
        pcm, n = inputs[w]
        pcm = np.ascontiguousarray(pcm, dtype=np.float32)
        last = {}
        for rep in range(args.repeats):
            for arm in arms:
                res, toks = run(pkg, model, arm, w, pcm, n)
                res.update(repeat=rep, gpu=gpu)
                print(json.dumps(res), flush=True)
                summary.setdefault((w, arm), []).append(res)
                last[arm] = toks
        for arm in arms[1:]:
            print(json.dumps({"workload": w, "tokens_new_vs_" + arm: agreement(last["new"], last[arm])}), flush=True)
    for (w, arm), rs in summary.items():
        x = [r["xRT"] for r in rs]
        print(json.dumps({"summary": w, "arm": arm, "gpu": gpu, "xRT": x, "xRT_mean": float(np.mean(x)), "rows_per_pass": rs[-1]["rows_per_pass"],
                          "decode_passes": rs[-1]["decode_passes"], "decode_gpu_ms_per_pass": [r["decode_gpu_ms_per_pass"] for r in rs]}), flush=True)


if __name__ == "__main__":
    main()

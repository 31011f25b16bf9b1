#!/usr/bin/env python3
"""The persistent decode kernel on the bench workload: partitions of a pass (WB200_MK_PARTS / WB200_MK_TURNS) and other builds, in one process.

Workload: the default line of bench.py -- large-v3 Q5_0 (synth.cached_model, seed 0), 64 x 30 s chunks, greedy, no timestamps, 224 tokens
per chunk, ONE whisper_full_parallel(ctx, params, pcm, n, 64) call per timed run (the first call of a context sizes its pool and is not timed).
Arms are given as name[:KEY=VALUE,...]; a key is an environment switch read when the context is created, or LIB=<path> for another build
of the same ABI.  Repeats alternate the arms (a, b, c, a, b, c, ...) so that the run-to-run spread is visible next to the differences.
Per run: xRT, decode passes, rows per pass, decode GPU ms per pass (wb200_counters [0]-[2]), encode GPU ms per window ([5], [6]), the card
and its power limit, and whether the token ids and probabilities of all chunks equal those of the first arm; the wall time no GPU work
covers (wall - passes x decode GPU ms - windows x encode GPU ms: host turnaround between passes) and the run-ahead rows launched and
taken (wb200_counters [12], [13]; a build without run-ahead reports zeros).
--trace ARM: one more, untimed run of that arm with WB200_MK_TRACE set; prints the per-phase split of a layer (us, CTA 0).

  python scripts/bench_decode.py --repeats 2 --arms parts1:WB200_MK_PARTS=1 parts2:WB200_MK_PARTS=2 parts4:WB200_MK_PARTS=4 \\
         parent:LIB=/path/to/parent/libwhisper_b200.so --trace parts1
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import load_pkg  # noqa: E402

DEFAULT_ARMS = ["parts1:WB200_MK_PARTS=1", "parts2:WB200_MK_PARTS=2", "parts4:WB200_MK_PARTS=4"]
LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_char_p, C.c_void_p)
QUIET = LOG_CB(lambda level, text, ud: None)


def parse_arm(text):
    """'name:K=V,K=V' -> (name, {K: V})"""
    name, _, rest = text.partition(":")
    env = {}
    for kv in filter(None, rest.split(",")):
        k, eq, v = kv.partition("=")
        if not eq or not k:
            raise ValueError(f"arm '{text}': expected KEY=VALUE, got '{kv}'")
        env[k] = v
    if not name:
        raise ValueError(f"arm '{text}' has no name")
    if "LIB" in env and not os.path.exists(env["LIB"]):
        raise FileNotFoundError(f"arm '{name}': {env['LIB']} does not exist")
    return name, env


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        lines = out.stdout.strip().splitlines() if out.returncode == 0 else []
    except (OSError, subprocess.SubprocessError):
        lines = []
    if not lines:
        raise SystemExit("no NVIDIA GPU: this script measures on the device and has nothing to fall back to")
    return lines[0]


def counters(L):
    a = (C.c_double * 14)(); L.wb200_counters(a, 14)
    return [a[i] for i in range(14)]


def outputs(L, ctx):
    """token ids and probabilities of all segments, in order"""
    ids, ps = [], []
    for s in range(L.whisper_full_n_segments(ctx)):
        for j in range(L.whisper_full_n_tokens(ctx, s)):
            ids.append(L.whisper_full_get_token_id(ctx, s, j)); ps.append(L.whisper_full_get_token_p(ctx, s, j))
    return np.array(ids, np.int64), np.array(ps, np.float32)


def run(pkg, model, env, pcm, n_chunks, trace=None):
    env = dict(env)
    lib = env.pop("LIB", pkg.LIB_PATH)
    if trace:
        env["WB200_MK_TRACE"] = trace
    os.environ.update(env)
    try:
        eng = pkg.WhisperB200(model, gpu_device=0, lib_path=lib)
    finally:
        for k in env:
            os.environ.pop(k, None)
    L = eng.L
    if not os.environ.get("WB200_VERBOSE"):
        L.whisper_log_set.argtypes = [LOG_CB, C.c_void_p]; L.whisper_log_set(QUIET, None)
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    L.whisper_full_get_token_p.restype = C.c_float
    p = L.whisper_full_default_params(0)
    p.print_progress = False; p.greedy.best_of = 1; p.temperature_inc = 0.0; p.no_timestamps = True; p.n_threads = 4
    buf = pcm.ctypes.data_as(C.c_void_p)
    call = lambda: L.whisper_full_parallel(eng.ctx, p, buf, len(pcm), n_chunks)  # noqa: E731
    assert call() == 0, L.wb200_last_error()
    c0 = counters(L)
    t0 = time.perf_counter()
    rc = call()
    dt = time.perf_counter() - t0
    c1 = counters(L)
    assert rc == 0, L.wb200_last_error()
    ids, ps = outputs(L, eng.ctx)
    eng.close()                                                  # the trace is written when the engine goes away
    passes = c1[0] - c0[0]
    gpu_ms = (c1[2] - c0[2]) + (c1[6] - c0[6])                       # decode passes + encoder windows, from their own events
    return {"xRT": len(pcm) / 16000.0 / dt, "wall_s": dt, "decode_passes": passes, "rows_per_pass": (c1[1] - c0[1]) / max(1.0, passes),
            "decode_gpu_ms_per_pass": (c1[2] - c0[2]) / max(1.0, passes), "encode_gpu_ms_per_window": (c1[6] - c0[6]) / max(1.0, c1[5] - c0[5]),
            "uncovered_ms": 1e3 * dt - gpu_ms, "uncovered_frac": 1.0 - gpu_ms / (1e3 * dt),
            "run_ahead_rows": c1[12] - c0[12], "run_ahead_taken": c1[13] - c0[13], "decoded_tokens": int(len(ids))}, ids, ps


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--chunks", type=int, default=64)
    ap.add_argument("--arms", nargs="+", default=DEFAULT_ARMS, metavar="NAME[:KEY=VALUE,...]")
    ap.add_argument("--trace", default=None, metavar="ARM", action="append", help="per-phase trace of this arm in an extra, untimed run (repeatable)")
    args = ap.parse_args()
    if args.repeats < 2:
        ap.error("--repeats must be at least 2: one run per arm says nothing about the spread")
    try:
        arms = [parse_arm(a) for a in args.arms]
    except (ValueError, FileNotFoundError) as e:
        ap.error(str(e))
    names = [n for n, _ in arms]
    for t in args.trace or []:
        if t not in names:
            ap.error(f"--trace {t}: no such arm")
    gpu = card()
    pkg = load_pkg(); synth = pkg.synth
    model = synth.cached_model("large-v3", synth.Q5_0, seed=0, fast_pool=True)
    pcm = np.ascontiguousarray(np.concatenate([synth.synth_audio(seed=i, seconds=30.0) for i in range(args.chunks)]), dtype=np.float32)
    first = None
    summary = {n: [] for n in names}
    for rep in range(args.repeats):
        for name, env in arms:
            res, ids, ps = run(pkg, model, env, pcm, args.chunks)
            if first is None:
                first = (ids, ps)
            res.update(arm=name, repeat=rep, gpu=gpu, same_tokens_as_first_arm=bool(np.array_equal(ids, first[0])),
                       same_probabilities_as_first_arm=bool(np.array_equal(ps.view(np.uint32), first[1].view(np.uint32))))
            print(json.dumps(res), flush=True)
            summary[name].append(res)
    for name in names:
        rs = summary[name]
        ms = [r["decode_gpu_ms_per_pass"] for r in rs]; x = [r["xRT"] for r in rs]
        print(json.dumps({"summary": name, "gpu": gpu, "decode_gpu_ms_per_pass": ms, "decode_gpu_ms_per_pass_mean": float(np.mean(ms)),
                          "uncovered_ms": [r["uncovered_ms"] for r in rs], "uncovered_frac": [r["uncovered_frac"] for r in rs],
                          "run_ahead_rows": [r["run_ahead_rows"] for r in rs], "run_ahead_taken": [r["run_ahead_taken"] for r in rs],
                          "encode_gpu_ms_per_window": [r["encode_gpu_ms_per_window"] for r in rs],
                          "xRT": x, "xRT_mean": float(np.mean(x)), "rows_per_pass": rs[-1]["rows_per_pass"], "decode_passes": rs[-1]["decode_passes"],
                          "same_as_first_arm": all(r["same_tokens_as_first_arm"] and r["same_probabilities_as_first_arm"] for r in rs)}), flush=True)
    for t in args.trace or []:
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "mk_trace.txt")
            run(pkg, model, dict(arms[names.index(t)][1]), pcm, args.chunks, trace=path)
            print(f"# trace of arm {t} ({gpu})")
            print(open(path).read() if os.path.exists(path) else "(this build wrote no trace)", flush=True)


if __name__ == "__main__":
    main()

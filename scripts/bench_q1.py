#!/usr/bin/env python3
"""Q5_1 models on their own kernels (this build) against the same file expanded to F16 at load time (the parent build, --parent-lib).

Models: synth.cached_model(<config>, Q5_1, seed=0, fast_pool=True) for small.en and base.en (the quantised downloads of these sizes are Q5_1).
Arms: `new` = this tree's library, `parent` = the library at --parent-lib (default $WB200_LIB), each run in a subprocess of its own;
repeats alternate the arms (new, parent, new, parent, ...) so that the run-to-run spread is visible next to the difference.
Workloads:
  a -- 64 x 30 s chunks, greedy, no timestamps, one whisper_full_parallel(ctx, p, pcm, n, 64) call (the shape of the default bench line)
  b -- --minutes of audio, greedy, one stream through whisper_full
  c -- the same audio, beam 5, one stream
Prints one JSON line per run (xRT, decode passes, rows per pass, decode GPU ms per pass, HBM image MB from the load log) and a summary per
(model, workload, arm); the card and its power limit come from nvidia-smi in the same call.

  python scripts/bench_q1.py --parent-lib /path/to/parent/libwhisper_b200.so [--repeats 2] [--minutes 3] [--workloads abc] [--models small.en,base.en]
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from __graft_entry__ import load_pkg  # noqa: E402

LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_char_p, C.c_void_p)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def counters(L):
    a = (C.c_double * 8)(); L.wb200_counters(a, 8)
    return [a[i] for i in range(8)]


def worker(lib_path, model, workload, minutes):
    """one timed run in this process; prints its JSON result"""
    pkg = load_pkg(); synth = pkg.synth
    log = []
    cb = LOG_CB(lambda level, text, ud: log.append(text.decode("utf-8", "replace")))
    raw = C.CDLL(lib_path)
    raw.whisper_log_set.argtypes = [LOG_CB, C.c_void_p]
    raw.whisper_log_set(cb, None)
    if workload == "a":
        pcm, n = np.concatenate([synth.synth_audio(seed=i, seconds=30.0) for i in range(64)]), 64
    else:
        pcm, n = np.concatenate([synth.synth_audio(seed=1234 + i, seconds=30.0) for i in range(max(1, int(round(minutes * 2))))]), 1
    pcm = np.ascontiguousarray(pcm, dtype=np.float32)
    eng = pkg.WhisperB200(model, gpu_device=0, lib_path=lib_path)
    L = eng.L
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    buf = pcm.ctypes.data_as(C.c_void_p)
    if workload == "c":
        p = L.whisper_full_default_params(1); p.beam_search.beam_size = 5
    else:
        p = L.whisper_full_default_params(0); p.greedy.best_of = 1
        p.no_timestamps = workload == "a"
    p.print_progress = False; p.temperature_inc = 0.0; p.n_threads = 4
    call = (lambda: L.whisper_full_parallel(eng.ctx, p, buf, len(pcm), n)) if n > 1 else (lambda: L.whisper_full(eng.ctx, p, buf, len(pcm)))
    assert call() == 0, L.wb200_last_error()                     # warm-up: sizes the context pool, loads every kernel the timed call uses
    c0 = counters(L)
    t0 = time.perf_counter()
    rc = call()
    dt = time.perf_counter() - t0
    c1 = counters(L)
    assert rc == 0, L.wb200_last_error()
    n_tok = sum(L.whisper_full_n_tokens(eng.ctx, s) for s in range(L.whisper_full_n_segments(eng.ctx)))
    eng.close()
    m = re.search(r"HBM image = ([0-9.]+) MB", "".join(log))
    passes = c1[0] - c0[0]
    print(json.dumps({"xRT": len(pcm) / 16000.0 / dt, "wall_s": dt, "decode_passes": passes, "rows_per_pass": (c1[1] - c0[1]) / max(1.0, passes),
                      "decode_gpu_ms_per_pass": (c1[2] - c0[2]) / max(1.0, passes), "decoded_tokens": n_tok,
                      "hbm_image_mb": float(m.group(1)) if m else None}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--parent-lib", default=os.environ.get("WB200_LIB"))
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--minutes", type=float, default=3.0, help="audio of workloads b and c")
    ap.add_argument("--workloads", default="abc")
    ap.add_argument("--models", default="small.en,base.en")
    ap.add_argument("--worker", nargs=3, metavar=("LIB", "MODEL", "WORKLOAD"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker(args.worker[0], args.worker[1], args.worker[2], args.minutes)
        return
    if not args.parent_lib or not os.path.exists(args.parent_lib):
        sys.exit("--parent-lib (or WB200_LIB): the parent build's libwhisper_b200.so is needed for the second arm")
    pkg = load_pkg(); synth = pkg.synth
    libs = {"new": os.path.join(ROOT, "whisper.cpp_b200", "libwhisper_b200.so"), "parent": os.path.abspath(args.parent_lib)}
    env = {k: v for k, v in os.environ.items() if k != "WB200_LIB"}
    gpu = card()
    summary = {}
    for cfg in args.models.split(","):
        model = synth.cached_model(cfg, synth.Q5_1, seed=0, fast_pool=True)
        for w in args.workloads:
            for rep in range(args.repeats):
                for arm, lib in libs.items():
                    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--minutes", str(args.minutes), "--worker", lib, model, w],
                                         capture_output=True, text=True, env=env, cwd=ROOT)
                    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
                    if out.returncode != 0 or not lines:
                        sys.exit("worker failed (%s, %s, %s):\n%s" % (cfg, w, arm, out.stderr[-3000:]))
                    res = json.loads(lines[-1])
                    res.update(model=cfg + " Q5_1", workload=w, arm=arm, repeat=rep, gpu=gpu)
                    print(json.dumps(res), flush=True)
                    summary.setdefault((cfg, w, arm), []).append(res)
    for (cfg, w, arm), rs in summary.items():
        x = [r["xRT"] for r in rs]
        print(json.dumps({"summary": cfg + " Q5_1", "workload": w, "arm": arm, "gpu": gpu, "xRT": x, "xRT_mean": float(np.mean(x)),
                          "decode_passes": rs[-1]["decode_passes"], "rows_per_pass": rs[-1]["rows_per_pass"],
                          "decode_gpu_ms_per_pass": [r["decode_gpu_ms_per_pass"] for r in rs], "hbm_image_mb": rs[-1]["hbm_image_mb"]}), flush=True)


if __name__ == "__main__":
    main()

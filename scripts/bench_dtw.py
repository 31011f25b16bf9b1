#!/usr/bin/env python3
"""DTW token timestamps at throughput: large-v3 Q5_0 with synthetic weights, `--chunks` x 30 s chunks, greedy, through ONE call of
whisper_full_parallel(ctx, params, pcm, n, n) -- the bench.py default workload (text-only decoding, 224 tokens per chunk) with
dtw_token_timestamps on (alignment heads: preset large-v3) or off.

One process measures one build (the library named by WB200_LIB, else the in-tree one); to compare builds, run the script once per build,
alternating, and compare the JSON lines.  Reported: x real time, decode passes and rows, the alignment-weight kernel's GPU time, the
device DTW path kernels' GPU time, the host DTW time (summed over the member threads), and the device->host bytes (wb200_traffic) -- with
DTW on they should exceed DTW off by the alignment-weight copies and the paths alone.  Counters a build does not have (k_dtw_qk time, host
DTW time, device DTW path time before they existed) read as 0.

  python scripts/bench_dtw.py --dtw on|off [--chunks 64] [--warmup 1] [--tag NAME]
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

LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_char_p, C.c_void_p)
QUIET = LOG_CB(lambda level, text, ud: None)
AHEADS_LARGE_V3 = 13                                     # WHISPER_AHEADS_LARGE_V3 (whisper.h)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtw", choices=("on", "off"), required=True)
    ap.add_argument("--chunks", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    pkg = load_pkg()
    synth = pkg.synth
    model = synth.cached_model("large-v3", synth.Q5_0, seed=0, fast_pool=True)
    L = pkg.bind_whisper_api(C.CDLL(pkg.LIB_PATH))
    L.whisper_log_set.argtypes = [LOG_CB, C.c_void_p]; L.whisper_log_set(QUIET, None)
    L.wb200_last_error.restype = C.c_char_p
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    L.wb200_traffic.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    cp = L.whisper_context_default_params()
    if args.dtw == "on":
        cp.flash_attn = False; cp.dtw_token_timestamps = True; cp.dtw_aheads_preset = AHEADS_LARGE_V3
    ctx = L.whisper_init_from_file_with_params(model.encode(), cp)
    if not ctx:
        raise SystemExit("context: " + L.wb200_last_error().decode())
    n = args.chunks
    pcm = np.ascontiguousarray(np.concatenate([synth.synth_audio(seed=i, seconds=30.0) for i in range(n)]), np.float32)
    p = L.whisper_full_default_params(0)
    p.print_progress = False; p.greedy.best_of = 1; p.temperature_inc = 0.0; p.no_timestamps = True; p.n_threads = 4

    def counters():
        a = (C.c_double * 16)(); L.wb200_counters(a, 16)
        h2d, d2h = C.c_uint64(), C.c_uint64(); L.wb200_traffic(C.byref(h2d), C.byref(d2h))
        return [a[i] for i in range(16)] + [float(h2d.value), float(d2h.value)]

    def run():
        rc = L.whisper_full_parallel(ctx, p, pcm.ctypes.data_as(C.c_void_p), len(pcm), n) if n > 1 else L.whisper_full(ctx, p, pcm.ctypes.data_as(C.c_void_p), len(pcm))
        if rc != 0:
            raise SystemExit("whisper_full_parallel: %d %s" % (rc, L.wb200_last_error().decode()))
    for _ in range(args.warmup):
        run()
    c0 = counters(); t0 = time.perf_counter()
    run()
    dt = time.perf_counter() - t0; c1 = counters()
    d = [b - a for a, b in zip(c0, c1)]
    n_tok = sum(L.whisper_full_n_tokens(ctx, i) for i in range(L.whisper_full_n_segments(ctx)))
    dtw_set = 0
    for i in range(L.whisper_full_n_segments(ctx)):
        for j in range(L.whisper_full_n_tokens(ctx, i)):
            dtw_set += L.whisper_full_get_token_data(ctx, i, j).t_dtw >= 0
    out = {"tag": args.tag, "lib": os.path.basename(os.path.dirname(pkg.LIB_PATH)) + "/" + os.path.basename(pkg.LIB_PATH), "dtw": args.dtw, "chunks": n,
           "audio_s": len(pcm) / 16000.0, "wall_s": round(dt, 3), "xRT": round(len(pcm) / 16000.0 / dt, 1), "tokens": n_tok, "tokens_with_t_dtw": dtw_set,
           "decode_passes": int(d[0]), "decode_rows": int(d[1]), "decode_gpu_ms": round(d[2], 1), "encode_windows": int(d[5]),
           "dtw_qk_gpu_ms": round(d[8], 2), "dtw_passes": int(d[9]), "dtw_path_gpu_ms": round(d[11], 2), "host_dtw_ms": round(d[10], 1), "h2d_bytes": int(d[16]), "d2h_bytes": int(d[17]),
           "card": card()}
    print(json.dumps(out), flush=True)
    L.whisper_free(ctx)


if __name__ == "__main__":
    main()

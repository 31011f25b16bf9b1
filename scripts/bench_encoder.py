#!/usr/bin/env python3
"""Time the batched encoder alone and split it by kernel role (large-v3 Q5_0 synthetic model, the bench.py default workload).

One process measures one build (the library named by WB200_LIB, else the in-tree one); to compare two builds, run the script once per
build, alternating, and compare the JSON lines.

  timed run     -- `--steps` lock-step batches of `--chunks` x 30 s chunks through wb200_full_batch_ex (device-resident PCM), after
                   `--warmup` batches; encode ms per window from the engine's CUDA-event counters (wb200_counters [5], [6])
  profiled run  -- one more batch under torch.profiler (CUDA activities): the encoder kernels in launch order, split by role.  Every
                   encoder GEMM is the same gemm_kernel symbol; a layer launches LayerNorm, qk, v, attention, o, LayerNorm, fc1, fc2, so the
                   role of a GEMM follows from its neighbours: the GEMMs in front of the first LayerNorm of an encode are conv1, conv2;
                   the two in front of the attention are qk, v; the one after it is o; the two after the next LayerNorm are fc1, fc2;
                   GEMMs after the final LayerNorm that no attention follows are the cross K/V
  outputs       -- one 30 s window through whisper_encode with WB200_DEBUG_TAPS=1: the encoder output (f32) and the cross K/V are
                   hashed (sha256 of the raw bytes) and the encoder output is written to OUT/enc_out.npy, for bit-for-bit comparisons

Prints one JSON line per phase and a summary line with TFLOP/s per role (algorithmic flops from the shapes over summed kernel time),
the card name and its power limit.

  python scripts/bench_encoder.py [--out DIR] [--tag NAME] [--steps 5] [--warmup 1] [--chunks 64] [--no-profile]
"""
import argparse
import ctypes as C
import hashlib
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

LOG_CB = C.CFUNCTYPE(None, C.c_int, C.c_char_p, C.c_void_p)
QUIET = LOG_CB(lambda level, text, ud: None)
ROLES = ("conv1", "conv2", "qk", "v", "attention", "o", "fc1", "fc2", "cross", "layernorm", "dequant", "other")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def kind(name):
    if "gemm_kernel" in name:
        return "gemm"
    if "fattn_enc_kernel" in name:
        return "attention"
    if "k_layernorm" in name:
        return "layernorm"
    if "k_dequant_f16" in name:
        return "dequant"
    return None


def split_roles(events):
    """events: [(kind, name, us)] of one stream in launch order, encoder kernels only (kind not None) -> {role: [us, launches]}.
    Encoder kernels of different encode calls are separated by None entries (a kernel of another kind in between)."""
    out = {r: [0.0, 0] for r in ROLES}

    def add(role, us):
        out[role][0] += us; out[role][1] += 1

    i, n = 0, len(events)
    after = "start"                                        # what the last LayerNorm followed: start / o / other
    last = "start"
    while i < n:
        ev = events[i]
        if ev is None:
            after = last = "start"; i += 1; continue
        k, us = ev[0], ev[2]
        if k == "layernorm":
            add("layernorm", us); after = "o" if last == "o" else "other"; last = "layernorm"; i += 1; continue
        if k == "dequant":
            add("dequant", us); i += 1; continue
        if k == "attention":
            add("attention", us); last = "attention"; i += 1; continue
        # a run of GEMMs (dequantisations in between skipped): its role follows from what is before and after it
        j, run = i, []
        while j < n and events[j] is not None and events[j][0] in ("gemm", "dequant"):
            if events[j][0] == "gemm":
                run.append(events[j][2])
            else:
                add("dequant", events[j][2])
            j += 1
        nxt = events[j][0] if j < n and events[j] is not None else None
        if last == "start":
            names = ["conv1", "conv2"] + ["other"] * (len(run) - 2)
        elif last == "attention":
            names = ["o"] * len(run)
        elif last == "layernorm" and after == "o":
            names = ["fc1", "fc2"] + ["other"] * (len(run) - 2)
        elif last == "layernorm" and nxt == "attention":
            names = ["qk", "v"] + ["other"] * (len(run) - 2)
        else:
            names = ["cross"] * len(run)
        for r, us in zip(names, run):
            add(r, us)
        last = names[-1] if names else last
        i = j
    return out


def role_flops(hp, n_win):
    """algorithmic flops of each role for n_win windows of n_audio_ctx frames (bench.py's encode_roofline, split)"""
    d, La, Lt, M, T = hp["n_audio_state"], hp["n_audio_layer"], hp["n_text_layer"], hp["n_mels"], hp["n_audio_ctx"]
    Tp = (T + 255) // 256 * 256
    f = {"conv1": 2 * 2 * T * 3 * M * d, "conv2": 2 * T * 3 * d * d, "qk": La * 2 * T * 2 * d * d, "v": La * 2 * T * d * d,
         "attention": La * 4 * T * Tp * d, "o": La * 2 * T * d * d, "fc1": La * 2 * T * 4 * d * d, "fc2": La * 2 * T * 4 * d * d,
         "cross": Lt * 2 * T * 2 * d * d}
    return {k: v * n_win for k, v in f.items()}


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def outputs(L, eng, synth, hp, out_dir, tag):
    """one 30 s window through whisper_encode on the context's own state: hashes of the encoder output and the cross K/V"""
    vp = C.c_void_p
    pcm0 = np.ascontiguousarray(synth.synth_audio(seed=0, seconds=30.0), dtype=np.float32)
    assert L.whisper_pcm_to_mel(eng.ctx, pcm0.ctypes.data_as(vp), len(pcm0), 1) == 0
    assert L.whisper_encode(eng.ctx, 0, 1) == 0, L.wb200_last_error()
    st0 = L.wb200_ctx_state(eng.ctx)
    hashes = {}
    for which, name in ((2, "encoder_out"), (3, "cross_k"), (4, "cross_v")):
        n = L.wb200_read_tensor(st0, which, None, 0)
        buf = np.empty(n, np.float32)
        assert L.wb200_read_tensor(st0, which, buf.ctypes.data_as(C.POINTER(C.c_float)), n) == n, L.wb200_last_error()
        hashes[name] = sha(buf)
        if which == 2:
            np.save(os.path.join(out_dir, "enc_out.npy"), buf.reshape(hp["n_audio_ctx"], hp["n_audio_state"]))
    print(json.dumps({"tag": tag, "phase": "outputs", "one_window_sha256": hashes}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=None, help="directory for enc_out.npy and the JSON lines (default: a temporary directory)")
    ap.add_argument("--tag", default=os.environ.get("WB200_LIB", "in-tree"))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--chunks", type=int, default=64)
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--outputs-only", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    out_dir = args.out or tempfile.mkdtemp(prefix="bench_encoder_")
    os.makedirs(out_dir, exist_ok=True)
    if not args.outputs_only:
        # the f32 encoder output needs WB200_DEBUG_TAPS, which adds work to every encode of the engine: a child process of its own
        env = dict(os.environ, WB200_DEBUG_TAPS="1")
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--outputs-only", "--out", out_dir, "--tag", args.tag], env=env,
                           capture_output=True, text=True)
        sys.stdout.write(r.stdout); sys.stderr.write(r.stderr[-4000:])
        assert r.returncode == 0, "outputs run failed"
        hashes = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])["one_window_sha256"]

    import torch
    pkg = load_pkg(); synth = pkg.synth
    if not os.environ.get("WB200_VERBOSE"):
        lib = C.CDLL(pkg.LIB_PATH)
        lib.whisper_log_set.argtypes = [LOG_CB, C.c_void_p]
        lib.whisper_log_set(QUIET, None)
    model = synth.cached_model("large-v3", synth.Q5_0, seed=0, fast_pool=True)
    gpu = card()
    eng = pkg.WhisperB200(model, gpu_device=0)
    L = eng.L
    vp = C.c_void_p
    L.wb200_counters.argtypes = [C.POINTER(C.c_double), C.c_int]
    L.wb200_full_batch_ex.argtypes = [vp, pkg.FullParams, C.POINTER(vp), C.POINTER(C.c_int), C.c_int, C.POINTER(vp), C.c_int]
    L.wb200_read_tensor.restype = C.c_int64
    L.wb200_read_tensor.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.c_int64]
    hp = {k: getattr(L, "whisper_model_" + k)(eng.ctx) for k in ("n_audio_state", "n_audio_layer", "n_text_layer", "n_mels", "n_audio_ctx")}

    def counters():
        a = (C.c_double * 8)(); L.wb200_counters(a, 8); return [a[i] for i in range(8)]

    if args.outputs_only:
        outputs(L, eng, synth, hp, out_dir, args.tag)
        eng.close()
        return

    # ---- batched encode, timed from the engine's CUDA events
    pcms = [torch.from_numpy(np.ascontiguousarray(synth.synth_audio(seed=i, seconds=30.0), dtype=np.float32)).cuda() for i in range(args.chunks)]
    p = L.whisper_full_default_params(0)
    p.print_progress = False; p.greedy.best_of = 1; p.temperature_inc = 0.0; p.no_timestamps = True; p.n_threads = 4
    n_arr = (C.c_int * args.chunks)(*[t.numel() for t in pcms])
    dev_ptrs = (vp * args.chunks)(*[t.data_ptr() for t in pcms])

    def batch():
        outs = (vp * args.chunks)()
        rc = L.wb200_full_batch_ex(eng.ctx, p, dev_ptrs, n_arr, args.chunks, outs, 1)
        assert rc == 0, (rc, L.wb200_last_error())
        for i in range(args.chunks):
            L.whisper_free_state(outs[i])

    for _ in range(args.warmup):
        batch()
    per_step = []
    for _ in range(args.steps):
        c0 = counters(); torch.cuda.synchronize(); t0 = time.perf_counter()
        batch()
        torch.cuda.synchronize(); dt = time.perf_counter() - t0; c1 = counters()
        per_step.append({"encode_ms_per_window": (c1[6] - c0[6]) / max(1.0, c1[5] - c0[5]), "encode_calls": c1[4] - c0[4],
                         "windows": c1[5] - c0[5], "step_s": dt})
    enc_ms = [s["encode_ms_per_window"] for s in per_step]
    print(json.dumps({"tag": args.tag, "phase": "timed", "gpu": gpu, "steps": per_step}), flush=True)

    res = {"tag": args.tag, "phase": "summary", "gpu": gpu, "chunks": args.chunks, "encode_ms_per_window": enc_ms,
           "encode_ms_per_window_median": float(np.median(enc_ms)), "one_window_sha256": hashes}
    # ---- one profiled batch: kernel times per role
    if not args.no_profile:
        from torch.profiler import ProfilerActivity, profile
        c0 = counters()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch()
            torch.cuda.synchronize()
        c1 = counters()
        n_win = c1[5] - c0[5]
        kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        kern.sort(key=lambda e: e.time_range.start)
        seq = []
        for e in kern:
            k = kind(e.name)
            if k is None:
                if seq and seq[-1] is not None and "k_mel" not in e.name and "k_zero_rows" not in e.name:
                    seq.append(None)                        # another kind of kernel between two encoder launches: a new encode
                continue
            seq.append((k, e.name, e.time_range.elapsed_us()))
        split = split_roles(seq)
        flops = role_flops(hp, n_win)
        total_us = sum(v[0] for v in split.values())
        roles = {}
        for r in ROLES:
            us, nl = split[r]
            if nl == 0:
                continue
            row = {"ms_per_window": us / 1e3 / max(1.0, n_win), "launches": nl, "share": us / max(total_us, 1e-9)}
            if r in flops and us > 0:
                row["TFLOPs"] = flops[r] / (us * 1e-6) / 1e12
            roles[r] = row
        gemm_us = sum(split[r][0] for r in ("conv1", "conv2", "qk", "v", "o", "fc1", "fc2", "cross"))
        gemm_fl = sum(flops[r] for r in ("conv1", "conv2", "qk", "v", "o", "fc1", "fc2", "cross"))
        res.update(profiled_windows=n_win, kernel_ms_per_window=total_us / 1e3 / max(1.0, n_win), roles=roles,
                   gemm_TFLOPs=gemm_fl / max(gemm_us * 1e-6, 1e-12) / 1e12)
    print(json.dumps(res), flush=True)
    with open(os.path.join(out_dir, "bench_encoder.json"), "a") as f:
        f.write(json.dumps(res) + "\n")
    eng.close()


if __name__ == "__main__":
    main()

"""Writes tests/golden/smoke_ref.npz: what __graft_entry__.smoke() compares against.

The unmodified reference CPU library (oracle/_ref/libwhisper_ref.so, built by __graft_entry__.build() from the reference tree) runs the
smoke input -- the synthetic 2-layer Q5_0 model (seed 7) on 5 s of synthetic audio (seed 1) -- through whisper_encode and three
whisper_decode steps (SOT, then the argmax token of each step).  Stored: the three decoded tokens and the logits of every step at a fixed,
seeded sample of 8192 vocabulary indices."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from __graft_entry__ import load_pkg, SMOKE_MODEL, SMOKE_AUDIO, SMOKE_STEPS, smoke_sample  # noqa: E402


def main(tmp="/tmp"):
    pkg = load_pkg(); synth = pkg.synth
    model = os.path.join(tmp, "smoke-q5_0.bin")
    synth.write_model(model, SMOKE_MODEL[0], synth.Q5_0, seed=SMOKE_MODEL[1])
    pcm = synth.synth_audio(seed=SMOKE_AUDIO[0], seconds=SMOKE_AUDIO[1])
    R = pkg.bind_whisper_api(C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libwhisper_ref.so")))
    cp = R.whisper_context_default_params(); cp.use_gpu = False
    ctx = R.whisper_init_from_file_with_params(model.encode(), cp)
    assert ctx
    assert R.whisper_pcm_to_mel(ctx, pcm.ctypes.data_as(C.c_void_p), len(pcm), 4) == 0
    assert R.whisper_encode(ctx, 0, 4) == 0
    n_vocab = R.whisper_n_vocab(ctx)
    idx = smoke_sample(n_vocab)
    tok = R.whisper_token_sot(ctx)
    tokens, logits = [], []
    for i in range(SMOKE_STEPS):
        t = np.array([tok], np.int32)
        assert R.whisper_decode(ctx, t.ctypes.data_as(C.c_void_p), 1, i, 4) == 0
        full = np.ctypeslib.as_array(R.whisper_get_logits(ctx), shape=(n_vocab,)).copy()
        tokens.append(tok); logits.append(full[idx])
        tok = int(full.argmax())
    R.whisper_free(ctx)
    out = os.path.join(ROOT, "tests", "golden", "smoke_ref.npz")
    np.savez_compressed(out, tokens=np.array(tokens, np.int32), index=idx, logits=np.array(logits, np.float32))
    print("wrote", out, "tokens", tokens)


if __name__ == "__main__":
    main()

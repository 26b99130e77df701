"""Determinism stress inside ONE process: the same prompt + forced decode steps, repeated N times with the KV cache cleared in
between; every repeat must give bit-identical logits.  Prints, per differing repeat, the first differing step.  Cheap enough
(tens of ms per repeat) to bisect rare races by configuration:

    python tools/stress_inproc.py small q4_k_m 200 GGML_B200_MEGA=0 GGML_B200_NO_GRAPHS=1
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
preset, ftype, n = sys.argv[1], sys.argv[2], int(sys.argv[3])
for kv in sys.argv[4:]:
    k, v = kv.split("=")
    os.environ[k] = v
os.environ["GGML_BACKEND_PATH"] = os.path.join(ROOT, "llama.cpp_b200", "libggml-b200.so")
gguf = f"/tmp/stress_{preset}_{ftype}.gguf"
if not os.path.exists(gguf):
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "make_gguf.py"), gguf, "--preset", preset, "--ftype", ftype])
L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "host", "libllama_host.so"))
L.lh_open.restype = C.c_void_p
L.lh_open.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]
L.lh_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
L.lh_n_vocab.argtypes = [C.c_void_p]
L.lh_clear.argtypes = [C.c_void_p]
L.lh_close.argtypes = [C.c_void_p]
n_prompt = int(os.environ.get("STRESS_PROMPT", "16"))
n_steps = int(os.environ.get("STRESS_STEPS", "6"))
h = L.lh_open(gguf.encode(), 99, 256, 64, 64, 1, 0, 8, None)
assert h
nv = L.lh_n_vocab(h)
toks = np.random.default_rng(7).integers(0, 512, size=max(n_prompt, n_steps)).astype(np.int32)


def once():
    out = []
    lp = np.empty(nv, np.float32)
    if n_prompt:
        assert L.lh_decode(h, toks.ctypes.data, n_prompt, lp.ctypes.data) == 0
        out.append(lp.copy())
    for t in toks[:n_steps]:
        one = np.array([t], np.int32)
        assert L.lh_decode(h, one.ctypes.data, 1, lp.ctypes.data) == 0
        out.append(lp.copy())
    return np.stack(out)


first = once()
bad = 0
first_steps = {}
for i in range(1, n):
    L.lh_clear(h)
    got = once()
    if not np.array_equal(first, got):
        bad += 1
        d = np.abs(got - first).max(axis=1)
        step = int(np.argmax(d > 0))
        first_steps[step] = first_steps.get(step, 0) + 1
        if bad <= 3:
            print(f"  repeat {i}: first differing step {step}, per-step max-abs {np.array2string(d, precision=3)}")
print(f"{preset}/{ftype} {' '.join(sys.argv[4:])}: {n} repeats, {bad} differing; first differing step histogram {first_steps}")
L.lh_close(h)

"""Multi-GPU check (run with gpurun --gpus N): -sm tensor through the reference's meta backend + our comm hooks.
Logits of a small random-init model: single GPU vs tensor-parallel over all visible GPUs, per all-reduce engine."""
import ctypes as C, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "llama.cpp_b200", "libggml-b200.so")
HOSTLIB = os.path.join(ROOT, "oracle", "_ref", "host", "libllama_host.so")
gguf = "/tmp/tp_small.gguf"
subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "make_gguf.py"), gguf, "--preset", "small", "--ftype", "q4_k_m"])
toks = np.random.default_rng(3).integers(0, 512, size=20)

def run(tag, sm, env_extra):
    code = f"""
import ctypes as C, numpy as np
L = C.CDLL({HOSTLIB!r})
L.lh_open.restype = C.c_void_p
L.lh_open.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]
L.lh_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
L.lh_n_vocab.argtypes = [C.c_void_p]
h = L.lh_open({gguf!r}.encode(), 99, 256, 64, 64, 1, {sm}, 8, None)
assert h
toks = np.array({toks.tolist()}, np.int32)
out = []
lp = np.empty(L.lh_n_vocab(h), np.float32)
assert L.lh_decode(h, toks.ctypes.data, len(toks), lp.ctypes.data) == 0
out.append(lp.copy())
for t in toks[:4]:
    one = np.array([int(t)], np.int32)
    assert L.lh_decode(h, one.ctypes.data, 1, lp.ctypes.data) == 0
    out.append(lp.copy())
np.save('/tmp/tp_{tag}.npy', np.stack(out))
"""
    env = dict(os.environ, GGML_BACKEND_PATH=PLUGIN)
    env.update(env_extra)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        print(tag, "FAILED rc", r.returncode, r.stderr[-1500:])
        return None
    for line in r.stderr.splitlines():
        if "ggml-b200" in line:
            print("   ", line)
    return np.load(f"/tmp/tp_{tag}.npy")

single = run("single", 0, {"CUDA_VISIBLE_DEVICES": "0"})
for tag, env in (("tp_default", {}), ("tp_nccl", {"GGML_B200_ALLREDUCE": "nccl"}), ("tp_oneshot", {"GGML_B200_ALLREDUCE": "oneshot"}),
                 ("tp_butterfly", {"GGML_B200_NO_COMM": "1"})):
    got = run(tag, 3, env)
    if got is None or single is None:
        continue
    print(f"{tag:>12}: max-abs vs single GPU {float(np.abs(got - single).max()):.3e}   max|logit| {float(np.abs(single).max()):.3f}  finite={bool(np.isfinite(got).all())}")

"""Diagnostic (GPU box): per-node comparison CPU vs GPU through llama's cb_eval hook, and logits error matrix."""
import ctypes as C, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ["GGML_BACKEND_PATH"] = os.path.join(ROOT, "llama.cpp_b200", "libggml-b200.so")
gguf = "/tmp/diag.gguf"
preset, ftype = (sys.argv[1:3] + ["small", "q4_k_m"])[:2] if len(sys.argv) >= 3 else ("small", "q4_k_m")
subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "make_gguf.py"), gguf, "--preset", preset, "--ftype", ftype])
toks = np.random.default_rng(7).integers(0, 512, size=24).astype(np.int32)

def run(tag, ngl, fa, dump, extra_env=None):
    env = dict(os.environ); env.update(extra_env or {})
    code = f"""
import ctypes as C, numpy as np, os
L = C.CDLL({os.path.join(ROOT, 'oracle', '_ref', 'host', 'libllama_host.so')!r})
L.lh_open.restype = C.c_void_p
L.lh_open.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]
L.lh_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
L.lh_n_vocab.argtypes = [C.c_void_p]
h = L.lh_open({gguf!r}.encode(), {ngl}, 256, 64, 64, {fa}, 0, 8, None)
toks = np.array({toks.tolist()}, np.int32)
lp = np.empty(L.lh_n_vocab(h), np.float32)
assert L.lh_decode(h, toks.ctypes.data, len(toks), lp.ctypes.data) == 0
np.save('/tmp/diag_{tag}.npy', lp)
"""
    if dump: env["LH_DUMP"] = f"/tmp/diag_{tag}.txt"
    subprocess.check_call([sys.executable, "-c", code], env=env)
    return np.load(f"/tmp/diag_{tag}.npy")

res = {}
res["cpu_fa1"] = run("cpu_fa1", 0, 1, True)
res["cpu_fa0"] = run("cpu_fa0", 0, 0, False)
res["gpu"] = run("gpu", 99, 1, True)
res["gpu_nofuse"] = run("gpu_nofuse", 99, 1, False, {"GGML_B200_NO_FUSION": "1", "GGML_B200_NO_GRAPHS": "1"})
print("max|logit| =", float(np.abs(res["cpu_fa1"]).max()))
keys = list(res)
for i, a in enumerate(keys):
    for b in keys[i + 1:]:
        print(f"{a:>12} vs {b:<12} max-abs {float(np.abs(res[a] - res[b]).max()):.3e}")
# per-node diff
def parse(path):
    out = []
    for line in open(path):
        p = line.split()
        if len(p) < 5 or not p[3].startswith("sum="): continue
        out.append((p[0], p[1], p[2], float(p[3][4:]), float(p[4][5:]), p[5] if len(p) > 5 else ""))
    return out
A, B = parse("/tmp/diag_cpu_fa1.txt"), parse("/tmp/diag_gpu.txt")
print(len(A), len(B), "nodes")
shown = 0
for a, b in zip(A, B):
    rel = abs(a[4] - b[4]) / (abs(a[4]) + 1e-30)
    flag = "  <<<<" if rel > 1e-3 else ""
    if shown < 60 or flag:
        print(f"{a[0]:>12} {a[1]:<22} {a[2]:<20} asum cpu={a[4]:.6g} gpu={b[4]:.6g} rel={rel:.2e}{flag}")
        shown += 1

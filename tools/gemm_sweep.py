"""GPU tuning aid: achieved TFLOP/s of the prefill GEMM (activation pre-pass + wgmma kernel) per shape."""
import json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import llama_cpp_b200.host as h  # noqa: E402
from tools.gemv_sweep import blocks, NAMES  # noqa: E402

def measure(t, M, K, N, gen):
    w = blocks(t, M, K, gen)
    x = torch.randn((N, K), device="cuda", generator=gen)
    out = torch.empty((N, M), device="cuda")
    ws = torch.empty(h.lib().b200_mul_mat_workspace_bytes(t, M, N, K), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        h.mul_mat(t, w, x, out=out, ws=ws)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        h.mul_mat(t, w, x, out=out, ws=ws)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return {"type": NAMES[t], "M": M, "K": K, "N": N, "ms": round(ms, 3), "TFLOPs": round(2.0 * M * N * K / ms / 1e9, 1)}

if __name__ == "__main__":
    gen = torch.Generator(device="cuda").manual_seed(0)
    for (t, M, K, N) in [(12, 4096, 4096, 512), (12, 4096, 4096, 2048), (12, 14336, 4096, 2048), (12, 4096, 14336, 2048), (14, 4096, 14336, 2048), (13, 4096, 4096, 2048), (2, 4096, 4096, 2048), (2, 11008, 4096, 2048), (8, 4096, 4096, 2048)]:
        try:
            print(json.dumps(measure(t, M, K, N, gen)), flush=True)
        except Exception as e:  # noqa: BLE001
            print(json.dumps({"type": NAMES[t], "M": M, "K": K, "N": N, "error": str(e).splitlines()[0]}), flush=True)

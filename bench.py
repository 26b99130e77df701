#!/usr/bin/env python
"""bench.py -- Llama-3-8B Q4_K_M decode (tg) through the drop-in boundary, on H100 (sm_90a).

Workload ("llama3-8b-q4_k_m-tg"): BASELINE.json configs[1].  A random-init Llama-3-8B GGUF with llama-quant.cpp's
Q4_K_M type mix (synthetic valid blocks, 4.91 GB; tools/make_gguf.py) is loaded by the REFERENCE's unmodified libllama
(oracle/_ref/host, built by oracle/host.mk) which dlopen()s our backend through GGML_BACKEND_PATH, exactly as llama-bench
would; one step = one decoded token (llama_decode of 1 token + llama_synchronize -- llama-bench's test_gen loop,
tools/llama-bench/llama-bench.cpp:2143-2162).  Every token streams the 4.6165 GB of mat-mul weights once
(SURVEY.md section 8d), far more than the 50 MB L2, so no L2 flush is needed between steps.

  value      tokens/s with everything resident on the device: the captured CUDA graph of one decode token is replayed
             K times between two CUDA events on the backend's stream (ggml_b200_replay_last_graph)
  e2e        tokens/s through the public API with HOST buffers: llama_decode() copies token id / position / KV indices /
             mask to the device and the 513 KB of logits back every step; wall clock around K steps, synchronised on
             both sides; h2d/d2h bytes are counted by the backend itself
  roofline   dominant kernel = decode_flow_kernel, the persistent dataflow decode kernel: ONE launch streams the whole token's
             4.6165 GB of mat-mul weights (32 layers + the output head), so the kernel IS the step; achieved = algorithmic bytes /
             the CUDA-event time of the replay; traffic = dram read+write of that launch from the committed ncu capture
             (profiles/r02_flow_ncu.json); none is committed, so it is null
  roofline_step   whole-token algorithmic bytes / device step time (the north-star's 0.70x target is this one)
  llama_bench     the reference's UNMODIFIED llama-bench (oracle/_ref/host/llama-bench -p 2048 -n 128 -ub 2048 -fa 1 -r 3) on the same
             GGUF through the same plugin, run after the timed region: the metric as SURVEY 8(d) defines it
  pp2048     prefill through the same API (llama-bench's test_prompt, -ub 2048) + the wgmma GEMM's achieved TFLOP/s
  cpu_baseline    the reference CPU backend (same libllama, n_gpu_layers = 0, all host threads) on a bounded sample

--dump-outputs DIR writes the logits of the last timed step (what llama_decode hands its caller for that token, re-read from
the device after the replay leg) as DIR/logits.npy, float32 [n_vocab].  The GGUF and the token ids are seeded, so two builds run
with the same arguments can be compared output for output.

N > 1: llama.cpp's tensor parallelism (-sm tensor, meta backend) is single-process: rank 0 drives all N GPUs through our
ggml_backend_comm_* hooks (default: one-shot NVLink all-reduce between per-GPU programs of the persistent kernel), the other
ranks only join the barriers (strong scaling, total work per token fixed).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
PLUGIN = os.path.join(ROOT, "llama.cpp_b200", "libggml-b200.so")
HOST_DIR = os.path.join(ROOT, "oracle", "_ref", "host")   # the reference's host programs + our driver over its API
HOSTLIB = os.path.join(HOST_DIR, "libllama_host.so")
ALG_BYTES_PER_TOKEN = 4.6165e9        # SURVEY.md section 8(d)
ALG_FLOP_PER_PP_TOKEN = 13.96e9
Q4_K = 12
N_CTX = 4096                          # both arms


def peaks():
    """(HBM GB/s, bf16 TFLOP/s burst, bf16 TFLOP/s sustained, source): data-sheet denominators unless measured peaks are given"""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        j = json.load(open(p))
        return float(j["hbm_gbs"]), float(j["bf16_tflops"]), float(j.get("bf16_tflops_sustained", j["bf16_tflops"])), "measured (MEASURED_PEAKS.json)"
    return 3350.0, 989.0, 989.0, "NVIDIA H100 SXM data sheet (dense, 700 W)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region (read-only queries)."""

    def __init__(self, index: int):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(self.index), "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm = sorted(int(r[0]) for r in self.rows if len(r) >= 6 and r[0].isdigit())
        mx = [int(r[1]) for r in self.rows if len(r) >= 6 and r[1].isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for r in self.rows if len(r) >= 6 for i in range(4) if r[2 + i].lower().startswith("active")})
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": reasons, "samples": len(sm)}


def gguf_path():
    d = "/dev/shm" if os.path.isdir("/dev/shm") and os.access("/dev/shm", os.W_OK) else "/tmp"
    return os.path.join(d, "b200-bench-llama3-8b-q4_k_m.gguf")


def ensure_gguf():
    p = gguf_path()
    if not (os.path.exists(p) and os.path.getsize(p) > 4.8e9):
        subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "make_gguf.py"), p, "--preset", "llama3-8b", "--ftype", "q4_k_m", "--quant", "synth"],
                              stdout=subprocess.DEVNULL)
    return p


def host_lib():
    if not os.path.exists(HOSTLIB):
        raise SystemExit(f"bench.py: {HOSTLIB} missing (run __graft_entry__.build() where the reference sources exist)")
    L = C.CDLL(HOSTLIB)
    L.lh_open.restype = C.c_void_p
    L.lh_open.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]
    L.lh_close.argtypes = [C.c_void_p]
    L.lh_clear.argtypes = [C.c_void_p]
    L.lh_test_gen.restype = C.c_double
    L.lh_test_gen.argtypes = [C.c_void_p, C.c_int, C.c_uint]
    L.lh_test_prompt.restype = C.c_double
    L.lh_test_prompt.argtypes = [C.c_void_p, C.c_int, C.c_uint]
    L.lh_n_vocab.argtypes = [C.c_void_p]
    L.lh_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return L


# ----------------------------------------------------------------------------------------------- reference / CPU leg
def cpu_reference(steps: int, warmup: int):
    """The reference's own CPU path for the same workload: same GGUF, same libllama, n_gpu_layers = 0, all host threads.
    Bounded sample: `steps` decoded tokens (each ~0.1-0.2 s on a server CPU)."""
    os.environ.pop("GGML_BACKEND_PATH", None)       # CPU only: do not even load the plugin
    L = host_lib()
    cores = os.cpu_count() or 1
    threads = min(cores, 64)
    h = L.lh_open(ensure_gguf().encode(), 0, N_CTX, 512, 512, 1, 0, threads, None)
    if not h:
        raise SystemExit("bench.py: reference CPU load failed")
    if warmup > 0:
        L.lh_test_gen(h, warmup, 1)
    L.lh_clear(h)
    sec = L.lh_test_gen(h, steps, 2)
    L.lh_close(h)
    return sec / steps, threads, f"{steps} decoded tokens of the same GGUF on the reference CPU backend (libllama, n_gpu_layers=0, {threads} threads), after {warmup} warm-up tokens"


def run_reference(args):
    if int(os.environ.get("RANK", "0")) != 0:
        return
    t0 = time.perf_counter()
    sec, threads, sample = cpu_reference(args.steps, args.warmup)
    val = 1.0 / sec
    print(json.dumps({
        "impl": "reference", "metric": "llama3-8b Q4_K_M tg tokens/s", "value": val, "unit": "tokens/s", "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "int8 x int4/6 -> int32, fp32 accumulate", "data": "synthetic random-init GGUF (Q4_K_M type mix), random token ids",
        "config": {"workload": "llama3-8b-q4_k_m-tg", "batch": 1, "n_ctx": N_CTX},
        "cpu_baseline": {"value": val, "unit": "tokens/s", "cores": threads, "kind": "reference", "sample": sample},
        "e2e": {"value": val, "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "wall_s": time.perf_counter() - t0}))


# ----------------------------------------------------------------------------------------------- dominant-kernel roofline
MEGA_DEFAULT = "1"                    # mirrors the plugin's default for GGML_B200_MEGA


def flow_traffic():
    """dram__bytes_read.sum + dram__bytes_write.sum of one decode_flow_kernel launch (one token), from the committed ncu --set full
    capture of the CURRENT kernel; None when there is none (never a number from another kernel version)."""
    p = os.path.join(ROOT, "profiles", "r02_flow_ncu.json")
    if not os.path.exists(p):
        return None, "no ncu capture of the current kernel committed yet"
    j = json.load(open(p))
    return float(j["dram_bytes_per_token"]), f"profiles/r02_flow_ncu.json ({j.get('note', '')})"


def llama_bench_leg(gguf):
    """The reference's unmodified llama-bench on the same GGUF through the same plugin (not inside the timed region)."""
    exe = os.path.join(HOST_DIR, "llama-bench")
    if not os.path.exists(exe):
        return {"unavailable": "oracle/_ref/host/llama-bench not built"}
    env = dict(os.environ, GGML_BACKEND_PATH=PLUGIN)
    try:
        out = subprocess.run([exe, "-m", gguf, "-p", "2048", "-n", "128", "-ub", "2048", "-fa", "1", "-r", "3", "-o", "jsonl"], env=env, capture_output=True, text=True, timeout=300)
    except subprocess.TimeoutExpired:
        return {"unavailable": "timeout"}
    res = {"cmd": "oracle/_ref/host/llama-bench -p 2048 -n 128 -ub 2048 -fa 1 -r 3 (GGML_BACKEND_PATH=libggml-b200.so)"}
    for ln in out.stdout.splitlines():
        try:
            j = json.loads(ln)
        except ValueError:
            continue
        key = f"pp{j['n_prompt']}" if j.get("n_prompt") else f"tg{j.get('n_gen')}"
        res[key] = {"tok_s": j.get("avg_ts"), "stddev": j.get("stddev_ts")}
    if len(res) == 1:
        res["unavailable"] = (out.stderr or out.stdout)[-300:]
    return res


def kernel_roofline():
    """gemv3_kernel<Q4_K> on the fused ffn_gate|ffn_up SwiGLU shape, cold weights, CUDA events around a graph of launches."""
    import torch
    import llama_cpp_b200.host as h
    gen = torch.Generator(device="cuda").manual_seed(1)
    M, K, nsets = 14336, 4096, 32
    rb = K // 256 * 144

    def blocks():
        w = torch.randint(0, 256, (M * rb + 16,), dtype=torch.uint8, device="cuda", generator=gen)
        v = w[: M * rb].view(M * (K // 256), 144)
        v[:, 1] = 0x0D
        v[:, 3] = 0x0D
        return w[: M * rb].view(M, rb)
    sets = [(blocks(), blocks()) for _ in range(nsets)]
    x = torch.randn(K, device="cuda", generator=gen)
    nw = torch.ones(K, device="cuda")
    outs = [torch.empty(M, device="cuda") for _ in range(nsets)]

    def go():
        for (g, u), o in zip(sets, outs):
            h.fused_matvec(Q4_K, [g, u], x, norm_w=nw, mode=2, outs=[o])
    go()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        go()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps / nsets
    nbytes = 2 * M * rb
    del sets
    torch.cuda.empty_cache()
    return nbytes, us


def gemm_tflops():
    import torch
    import llama_cpp_b200.host as h
    gen = torch.Generator(device="cuda").manual_seed(2)
    M, K, N = 14336, 4096, 2048
    rb = K // 256 * 144
    w = torch.randint(0, 256, (M * rb + 16,), dtype=torch.uint8, device="cuda", generator=gen)
    v = w[: M * rb].view(M * (K // 256), 144)
    v[:, 1] = 0x0D
    v[:, 3] = 0x0D
    w = w[: M * rb].view(M, rb)
    x = torch.randn((N, K), device="cuda", generator=gen)
    out = torch.empty((N, M), device="cuda")
    ws = torch.empty(h.lib().b200_mul_mat_workspace_bytes(Q4_K, M, N, K), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        h.mul_mat(Q4_K, w, x, out=out, ws=ws)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        h.mul_mat(Q4_K, w, x, out=out, ws=ws)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    return 2.0 * M * N * K / ms / 1e9, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="b200")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-pp", action="store_true")
    ap.add_argument("--no-llama-bench", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's logits to DIR/logits.npy (float32)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    if args.dump_outputs and args.gpus != 1:
        ap.error("--dump-outputs needs --gpus 1 (the logits are re-read after the single-GPU replay leg)")
    if args.impl == "reference":
        return run_reference(args)

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}: launch N>1 with torch.distributed.run"
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("gloo")
        if rank != 0:                  # llama.cpp's tensor parallelism is single-process: rank 0 drives all GPUs
            dist.barrier()
            dist.barrier()
            dist.destroy_process_group()
            return

    if not os.path.exists(PLUGIN):
        raise SystemExit(f"bench.py: {PLUGIN} missing -- refusing to fall back to anything else")
    os.environ["GGML_BACKEND_PATH"] = PLUGIN
    L = host_lib()                     # first: it loads the host's libggml-base.so, which the plugin names by soname
    plug = C.CDLL(PLUGIN, mode=C.RTLD_GLOBAL)
    plug.ggml_backend_score.restype = C.c_int
    if plug.ggml_backend_score() <= 0:
        raise SystemExit("bench.py: the backend reports no usable sm_90 device -- refusing to fall back to anything else")
    plug.ggml_b200_replay_last_graph.argtypes = [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_ulonglong)]
    plug.ggml_b200_stats.argtypes = [C.POINTER(C.c_ulonglong)] * 3
    plug.ggml_b200_reread_last_output.restype = C.c_ulonglong
    plug.ggml_b200_reread_last_output.argtypes = [C.c_void_p, C.c_ulonglong]
    plug.ggml_b200_enable_replay(1)

    def stats():
        a, b, c = C.c_ulonglong(), C.c_ulonglong(), C.c_ulonglong()
        plug.ggml_b200_stats(C.byref(a), C.byref(b), C.byref(c))
        return a.value, b.value, c.value

    W = max(3, args.warmup)
    K = args.steps
    devs = ",".join(f"B200{i}" for i in range(world)).encode() if world > 1 else None
    h = L.lh_open(ensure_gguf().encode(), 99, N_CTX, 2048, 2048, 1, 3 if world > 1 else 0, 8, devs)
    if not h:
        raise SystemExit("bench.py: model load through the plugin failed")

    # ---- e2e leg: llama_decode + llama_synchronize per token, host buffers in and out (llama-bench's test_gen)
    L.lh_test_gen(h, W, 1)
    L.lh_clear(h)
    L.lh_test_gen(h, W, 2)             # leave W tokens in the cache so the timed steps run at a realistic short context
    sampler = ClockSampler(0)
    sampler.start()
    h2d0, d2h0, l0 = stats()
    if dist:
        dist.barrier()
    sec_e2e = L.lh_test_gen(h, K, 3)
    h2d1, d2h1, l1 = stats()
    tok_s_e2e = K / sec_e2e

    mega_on = os.environ.get("GGML_B200_MEGA", MEGA_DEFAULT) not in ("", "0")
    # ---- device-resident leg: replay the captured decode graph between CUDA events (single GPU only)
    ms = C.c_float(0)
    per = C.c_ulonglong(0)
    have_replay = world == 1 and plug.ggml_b200_replay_last_graph(W, C.byref(ms), C.byref(per)) == 0
    replay_check = None
    if have_replay:
        # what the replays compute must be what the end-to-end step computed: the replay restores the inputs of the LAST decoded token,
        # so its logits (re-read from the device region llama_decode read them from) must equal that step's logits bit for bit
        import numpy as np
        nv = L.lh_n_vocab(h)
        host_logits = np.empty(nv, np.float32)
        tok = np.array([12345 % nv], np.int32)
        if L.lh_decode(h, tok.ctypes.data, 1, host_logits.ctypes.data) != 0:
            raise SystemExit("bench.py: llama_decode failed")
        plug.ggml_b200_replay_last_graph(2, C.byref(ms), C.byref(per))
        dev_logits = np.empty(nv, np.float32)
        got = plug.ggml_b200_reread_last_output(dev_logits.ctypes.data, C.c_ulonglong(dev_logits.nbytes))
        if not np.isfinite(host_logits).all():
            raise SystemExit("bench.py: non-finite logits from the end-to-end step")
        replay_check = {"bytes": int(got), "finite": bool(np.isfinite(dev_logits).all()) if got else None,
                        "same_argmax": bool(int(dev_logits.argmax()) == int(host_logits.argmax())) if got else None,
                        "bit_identical": bool(np.array_equal(dev_logits, host_logits)) if got else None}
        if got and not (replay_check["finite"] and replay_check["same_argmax"]):
            raise SystemExit(f"bench.py: the replayed graph does not reproduce the end-to-end step's logits: {replay_check}")
        plug.ggml_b200_replay_last_graph(K, C.byref(ms), C.byref(per))
        ms_dev = float(ms.value)
        if args.dump_outputs:
            last = np.empty(nv, np.float32)
            if plug.ggml_b200_reread_last_output(last.ctypes.data, C.c_ulonglong(last.nbytes)) != last.nbytes:
                raise SystemExit("bench.py: could not re-read the last timed step's logits")
            os.makedirs(args.dump_outputs, exist_ok=True)
            np.save(os.path.join(args.dump_outputs, "logits.npy"), last)
        tok_s = K / (ms_dev * 1e-3)
        launches = int(per.value) * K
    else:
        ms_dev = sec_e2e * 1e3
        tok_s = tok_s_e2e
        launches = l1 - l0
        if args.dump_outputs:
            sampler.stop()
            raise SystemExit("bench.py: --dump-outputs needs the single-GPU replay leg")
    clocks = sampler.stop()

    # ---- prefill pp2048 through the same API
    pp = None
    if not args.no_pp:
        L.lh_clear(h)
        L.lh_test_prompt(h, 2048, 5)
        L.lh_clear(h)
        s_pp = 1e30
        for i in range(2):
            L.lh_clear(h)
            s_pp = min(s_pp, L.lh_test_prompt(h, 2048, 6 + i))
        pp = {"value": 2048 / s_pp, "unit": "tokens/s", "n_prompt": 2048, "n_ubatch": 2048, "ms": s_pp * 1e3}
    L.lh_close(h)
    if dist:
        dist.barrier()

    hbm_peak, tf_burst, tf_peak, peak_src = peaks()
    line = {
        "metric": "llama3-8b Q4_K_M tg tokens/s", "value": tok_s, "unit": "tokens/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": ms_dev / K, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "int8 x int4/6 -> int32, fp32 accumulate", "data": "synthetic random-init GGUF (Q4_K_M type mix), random token ids",
        "config": {"workload": "llama3-8b-q4_k_m-tg", "batch": 1, "n_ctx": 4096, "kv_tokens_during_timing": f"{W}..{W + K}",
                   "host": "reference libllama (oracle/_ref/host) + GGML_BACKEND_PATH=libggml-b200.so", "flash_attn": True,
                   "parallelism": f"-sm tensor x{world} (meta backend + ggml_backend_comm_* hooks)" if world > 1 else "single GPU",
                   "l2": "4.6 GB of weights streamed per step, larger than L2; no flush needed",
                   # N = 1: the captured graph of one token is what the replay leg times.  N > 1: every per-GPU segment between two all-reduces
                   # is captured and replayed by graph uid inside the plugin; the device-replay hook itself is single-GPU, so value = e2e there
                   "cuda_graph": bool(have_replay) if world == 1 else "per-GPU segments captured by graph uid (plugin); no whole-token replay leg",
                   "decode_kernel": "persistent dataflow kernel (decode_flow.cu)" if mega_on else "one fused launch per mat-vec group (gemv3.cu)"},
        "clocks": clocks, "gpu_launches": launches,
        "e2e": {"value": tok_s_e2e, "unit": "tokens/s", "h2d_bytes_per_step": (h2d1 - h2d0) // K, "d2h_bytes_per_step": (d2h1 - d2h0) // K,
                "timing": "wall clock around K x (llama_decode + llama_synchronize)"},
        "roofline_step": {"bound": "hbm", "achieved": ALG_BYTES_PER_TOKEN / world * tok_s / 1e9, "peak": hbm_peak, "unit": "GB/s",
                          "frac": ALG_BYTES_PER_TOKEN / world * tok_s / 1e9 / hbm_peak, "bytes_per_token_per_gpu": ALG_BYTES_PER_TOKEN / world},
    }
    if pp:
        line["pp2048"] = pp
    if replay_check is not None:
        line["replay_check"] = replay_check
    if world == 1:
        nbytes, us = kernel_roofline()
        ach = nbytes / us / 1e3
        gemv3 = {"bound": "hbm", "kernel": "gemv3_kernel<Q4_K> fused RMS_NORM+Q8_K+ffn_gate|ffn_up+SwiGLU, 2x14336x4096", "achieved": ach, "peak": hbm_peak,
                 "unit": "GB/s", "frac": ach / hbm_peak, "traffic": None, "peak_source": peak_src, "bytes_per_launch": nbytes, "us_per_launch": us}
        if mega_on and have_replay:
            # the persistent decode kernel IS the step: one launch streams the whole token's weights (plus 2 tiny launches: the
            # token-embedding GET_ROWS on quantised rows and the replay's input restore), timed live by the CUDA events of the replay
            us_tok = ms_dev * 1e3 / K
            ach = ALG_BYTES_PER_TOKEN / us_tok / 1e3
            traffic, traffic_src = flow_traffic()
            line["roofline"] = {"bound": "hbm", "kernel": "decode_flow_kernel (persistent dataflow kernel: one launch per token, all 32 layers + final norm + head)", "achieved": ach,
                                "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak, "traffic": traffic, "peak_source": peak_src,
                                "bytes_per_launch": ALG_BYTES_PER_TOKEN, "us_per_launch": us_tok, "traffic_source": traffic_src}
            line["matvec_kernel_roofline"] = gemv3
        else:
            line["roofline"] = gemv3
        if pp:
            tf, ms_g = gemm_tflops()
            # the GEMM is timed alone over a few ms: the BURST cuBLAS figure is its denominator; the pp2048 step runs ~100 ms inside a
            # longer job: the SUSTAINED figure is its denominator.  Both fractions are given for both.
            pp["gemm_roofline"] = {"bound": "tensor", "kernel": "gemm_q_wgmma Q4_K 14336x2048x4096 (+ activation pre-pass)", "achieved": tf,
                                   "peak": tf_burst, "unit": "TFLOP/s", "frac": tf / tf_burst, "frac_of_sustained": tf / tf_peak, "ms_per_launch": ms_g,
                                   "peak_kind": "burst"}
            ach_pp = ALG_FLOP_PER_PP_TOKEN * pp["value"] / 1e12
            pp["roofline_step"] = {"bound": "tensor", "achieved": ach_pp, "peak": tf_peak, "unit": "TFLOP/s", "frac": ach_pp / tf_peak,
                                   "frac_of_burst": ach_pp / tf_burst, "peak_kind": "sustained"}
    if world == 1 and not args.no_llama_bench:
        line["llama_bench"] = llama_bench_leg(gguf_path())
    if not args.no_cpu_baseline:
        sec, threads, sample = cpu_reference(8, 2)
        line["cpu_baseline"] = {"value": 1.0 / sec, "unit": "tokens/s", "cores": threads, "kind": "reference", "sample": sample}
    print(json.dumps(line))
    if dist:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

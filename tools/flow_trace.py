"""Phase timeline of the persistent decode kernel (csrc/decode_flow.cu) at the benchmark's workload.

Loads the bench GGUF (bench.py's Llama-3-8B Q4_K_M, made by tools/make_gguf.py if missing) through the reference's libllama
(the host programs build() makes) with our plugin, exactly as bench.py opens it, decodes bench.py's two rounds of 8 warm-up tokens and then
--tokens more, with GGML_B200_MEGA_TRACE set.  The plugin dumps the last decode launch's per-phase, per-CTA globaltimer stamps
when the context is freed; tools/mega_trace.py summarises them.  Writes OUT (markdown): the GPU's name, power limit and
maximum SM clock read in the same run, the command, and the summary.

    python tools/flow_trace.py profiles/h100_flow_trace.md [--tokens 16]
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the benchmark's GGUF, host library and context parameters)


def gpu_info() -> str:
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    except OSError as e:
        raise SystemExit(f"flow_trace.py: needs a GPU and nvidia-smi ({e})")
    if out.returncode != 0:
        raise SystemExit(f"flow_trace.py: nvidia-smi failed: {out.stderr.strip()}")
    name, power, sm_max, driver = (c.strip() for c in out.stdout.strip().split(","))
    return f"{name}, power limit {power}, max SM clock {sm_max}, driver {driver}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", help="markdown summary to write")
    ap.add_argument("--tokens", type=int, default=16, help="tokens decoded after the warm-up; the last one is traced")
    ap.add_argument("--title", default="Phase trace of the persistent decode kernel")
    args = ap.parse_args()
    if args.tokens < 1:
        ap.error("--tokens must be >= 1")
    if not os.path.exists(bench.PLUGIN):
        raise SystemExit(f"flow_trace.py: {bench.PLUGIN} missing (run __graft_entry__.build())")
    info = gpu_info()
    gguf = bench.ensure_gguf()
    warm = 8
    with tempfile.TemporaryDirectory() as td:
        dump = os.path.join(td, "flow_trace.bin")
        os.environ["GGML_BACKEND_PATH"] = bench.PLUGIN
        os.environ["GGML_B200_MEGA_TRACE"] = dump
        L = bench.host_lib()
        h = L.lh_open(gguf.encode(), 99, bench.N_CTX, 2048, 2048, 1, 0, 8, None)
        if not h:
            raise SystemExit("flow_trace.py: model load through the plugin failed")
        L.lh_test_gen(h, warm, 1)                # bench.py's warm-up: W tokens, clear, W tokens left in the cache
        L.lh_clear(h)
        L.lh_test_gen(h, warm, 2)
        if L.lh_test_gen(h, args.tokens, 3) < 0:
            raise SystemExit("flow_trace.py: llama_decode failed")
        L.lh_close(h)                            # frees the backend: the plugin writes the dump
        if not os.path.exists(dump):
            raise SystemExit("flow_trace.py: the plugin wrote no trace (is the persistent decode kernel on?)")
        summary = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "mega_trace.py"), dump], capture_output=True, text=True, check=True).stdout
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(f"# {args.title}\n\n")
        f.write(f"GPU: {info}.\n\n")
        f.write(f"`python tools/flow_trace.py {os.path.basename(args.out)} --tokens {args.tokens}`: bench.py's GGUF and context (n_ctx {bench.N_CTX}), "
                f"{warm} + {warm} warm-up tokens, then {args.tokens} decoded; the last one ({warm + args.tokens} tokens in the cache) is traced.  "
                f"Summary by tools/mega_trace.py.\n\n")
        f.write("```\n" + summary + "```\n")
    print(open(args.out).read())


if __name__ == "__main__":
    main()

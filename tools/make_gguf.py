#!/usr/bin/env python
"""Random-init Llama/Mixtral GGUF files for the parity harness and the benchmark (SURVEY.md section 8d recipe).

  --quant exact   weights ~ N(0, 0.02) quantised per tensor by the REFERENCE quantiser (ggml_quantize_chunk of the reference
                  host's own libggml-base.so, found on LD_LIBRARY_PATH -- what llama-quantize calls per tensor)
                  with llama-quant.cpp's Q4_K_M / Q5_K_M / Q4_0 type mix -- for logits parity on small models
  --quant synth   random valid blocks written directly (no f32 weights, no quantiser) -- for 8B/70B-sized bench files

No tokenizer is stored (tokenizer.ggml.model = "no_vocab"); prompts are token ids.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gguf  # noqa: E402
from gguf import GGMLQuantizationType as QT  # noqa: E402

# enum ggml_type values (ggml/include/ggml.h:388-410) and block geometry (ggml-common.h:194-376).  Self-contained on purpose: this
# tool writes bench / test DATA and is run by bench.py, which must not execute anything under oracle/ outside its CPU legs.
Q4_0, Q8_0, Q4_K, Q5_K, Q6_K = 2, 8, 12, 13, 14
BLOCK_ELEMS = {Q4_0: 32, Q8_0: 32, Q4_K: 256, Q5_K: 256, Q6_K: 256}
BLOCK_BYTES = {Q4_0: 18, Q8_0: 34, Q4_K: 144, Q5_K: 176, Q6_K: 210}


def random_blocks(t, rows, k, rng, scale=0.02):
    """Random but VALID quantised rows (uint8 [rows, row_bytes]): random codes and sub-scales, fp16 super-scales sized so that
    the dequantised weights are O(scale).  No quantiser involved (an 8B file takes seconds, not minutes)."""
    nb, bb = k // BLOCK_ELEMS[t], BLOCK_BYTES[t]
    out = rng.integers(0, 256, size=(rows, nb, bb), dtype=np.uint8)

    def put_half(off, vals):
        h = np.asarray(vals, dtype=np.float16).view(np.uint16)
        out[:, :, off] = (h & 0xFF).astype(np.uint8)
        out[:, :, off + 1] = (h >> 8).astype(np.uint8)

    u = rng.uniform(0.5, 1.0, size=(rows, nb))
    if t == Q4_0:
        put_half(0, u * scale / 4)
    elif t == Q8_0:
        put_half(0, u * scale / 64)
    elif t in (Q4_K, Q5_K):
        put_half(0, u * scale / (32 * (15 if t == Q4_K else 31)) * 4)
        put_half(2, rng.uniform(0.5, 1.0, size=(rows, nb)) * scale / 32)
    else:
        put_half(208, u * scale / (64 * 32) * 2)
    return out.reshape(rows, nb * bb)


class HostQuantiser:
    """ggml_quantize_chunk (ggml/src/ggml.c) from the reference host's libggml-base.so (the one the dynamic loader finds)."""

    def __init__(self):
        import ctypes as C
        self.C = C
        self.lib = C.CDLL("libggml-base.so")
        self.lib.ggml_quantize_chunk.restype = C.c_size_t
        self.lib.ggml_quantize_chunk.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]

    def quantize_weights(self, t, w):
        w = np.ascontiguousarray(w, dtype=np.float32)
        M, K = w.shape
        out = np.empty((M, K // BLOCK_ELEMS[t] * BLOCK_BYTES[t]), dtype=np.uint8)
        n = self.lib.ggml_quantize_chunk(t, w.ctypes.data, out.ctypes.data, 0, M, K, None)
        assert n == out.size
        return out

QT_OF = {Q4_0: QT.Q4_0, Q8_0: QT.Q8_0, Q4_K: QT.Q4_K, Q5_K: QT.Q5_K, Q6_K: QT.Q6_K}
PRESETS = {
    "tiny":       dict(n_embd=256, n_ff=512, n_head=4, n_head_kv=2, n_layer=2, n_vocab=512),
    "small":      dict(n_embd=1024, n_ff=2816 // 256 * 256, n_head=8, n_head_kv=4, n_layer=4, n_vocab=4096),
    "llama3-8b":  dict(n_embd=4096, n_ff=14336, n_head=32, n_head_kv=8, n_layer=32, n_vocab=128256, rope_base=500000.0),
    "llama2-7b":  dict(n_embd=4096, n_ff=11008, n_head=32, n_head_kv=32, n_layer=32, n_vocab=32000),
    "llama3-70b": dict(n_embd=8192, n_ff=28672, n_head=64, n_head_kv=8, n_layer=80, n_vocab=128256, rope_base=500000.0),
    "mixtral-8x7b": dict(n_embd=4096, n_ff=14336, n_head=32, n_head_kv=8, n_layer=32, n_vocab=32000, n_expert=8, n_expert_used=2, rope_base=1000000.0),
    "tiny-moe":   dict(n_embd=256, n_ff=512, n_head=4, n_head_kv=2, n_layer=2, n_vocab=512, n_expert=4, n_expert_used=2),
}


def more_bits(i, n):
    return i < n // 8 or i >= 7 * n // 8 or (i - n // 8) % 3 == 2


def tensor_type(ftype, name, i, n_layer):
    """Type mix of llama-quant.cpp:430-475,552-619 for the tensors a Llama/Mixtral model has."""
    if ftype == "q4_0":
        return Q6_K if name == "output" else Q4_0
    if ftype == "q8_0":
        return Q8_0
    base, hi = (Q4_K, Q6_K) if ftype == "q4_k_m" else (Q5_K, Q6_K)
    if name in ("output", "token_embd"):
        return hi if name == "output" else base
    if name in ("attn_v", "ffn_down", "ffn_down_exps") and more_bits(i, n_layer):
        return hi
    return base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--preset", default="tiny", choices=sorted(PRESETS))
    ap.add_argument("--ftype", default="q4_k_m", choices=["q4_k_m", "q5_k_m", "q4_0", "q8_0"])
    ap.add_argument("--quant", default="exact", choices=["exact", "synth"])
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--ctx", type=int, default=4096)
    ap.add_argument("--layers", type=int, default=0, help="override n_layer")
    args = ap.parse_args()
    hp = dict(PRESETS[args.preset])
    if args.layers:
        hp["n_layer"] = args.layers
    n_embd, n_ff, n_head, n_head_kv, n_layer, n_vocab = (hp[k] for k in ("n_embd", "n_ff", "n_head", "n_head_kv", "n_layer", "n_vocab"))
    n_expert = hp.get("n_expert", 0)
    head_dim = n_embd // n_head
    rng = np.random.default_rng(args.seed)
    ref = None
    if args.quant == "exact":
        ref = HostQuantiser()

    w = gguf.GGUFWriter(args.out, "llama")
    w.add_vocab_size(n_vocab)
    w.add_context_length(args.ctx)
    w.add_embedding_length(n_embd)
    w.add_block_count(n_layer)
    w.add_feed_forward_length(n_ff)
    w.add_head_count(n_head)
    w.add_head_count_kv(n_head_kv)
    w.add_layer_norm_rms_eps(1e-5)
    w.add_rope_dimension_count(head_dim)
    if "rope_base" in hp:
        w.add_rope_freq_base(hp["rope_base"])
    if n_expert:
        w.add_expert_count(n_expert)
        w.add_expert_used_count(hp["n_expert_used"])
    w.add_tokenizer_model("no_vocab")
    w.add_file_type({"q4_k_m": 15, "q5_k_m": 17, "q4_0": 2, "q8_0": 7}[args.ftype])

    def qtensor(name, short, i, rows, k, experts=0):
        t = tensor_type(args.ftype, short, i, n_layer)
        ne = max(experts, 1)
        if ref is not None:
            f = (rng.standard_normal((ne * rows, k)) * 0.02).astype(np.float32)
            data = ref.quantize_weights(t, f)
        else:
            data = random_blocks(t, ne * rows, k, rng)
        shape = [ne, rows, data.shape[1]] if experts else [rows, data.shape[1]]
        w.add_tensor(name, data.reshape(shape), raw_dtype=QT_OF[t])

    def f32tensor(name, arr):
        w.add_tensor(name, arr.astype(np.float32))

    qtensor("token_embd.weight", "token_embd", 0, n_vocab, n_embd)
    f32tensor("output_norm.weight", 1.0 + 0.1 * rng.standard_normal(n_embd))
    qtensor("output.weight", "output", 0, n_vocab, n_embd)
    for i in range(n_layer):
        p = f"blk.{i}."
        f32tensor(p + "attn_norm.weight", 1.0 + 0.1 * rng.standard_normal(n_embd))
        qtensor(p + "attn_q.weight", "attn_q", i, n_head * head_dim, n_embd)
        qtensor(p + "attn_k.weight", "attn_k", i, n_head_kv * head_dim, n_embd)
        qtensor(p + "attn_v.weight", "attn_v", i, n_head_kv * head_dim, n_embd)
        qtensor(p + "attn_output.weight", "attn_output", i, n_embd, n_head * head_dim)
        f32tensor(p + "ffn_norm.weight", 1.0 + 0.1 * rng.standard_normal(n_embd))
        if n_expert:
            f32tensor(p + "ffn_gate_inp.weight", rng.standard_normal((n_expert, n_embd)) * 0.02)
            qtensor(p + "ffn_gate_exps.weight", "ffn_gate_exps", i, n_ff, n_embd, n_expert)
            qtensor(p + "ffn_down_exps.weight", "ffn_down_exps", i, n_embd, n_ff, n_expert)
            qtensor(p + "ffn_up_exps.weight", "ffn_up_exps", i, n_ff, n_embd, n_expert)
        else:
            qtensor(p + "ffn_gate.weight", "ffn_gate", i, n_ff, n_embd)
            qtensor(p + "ffn_down.weight", "ffn_down", i, n_embd, n_ff)
            qtensor(p + "ffn_up.weight", "ffn_up", i, n_ff, n_embd)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    print(f"wrote {args.out}: {os.path.getsize(args.out) / 1e6:.1f} MB  preset={args.preset} ftype={args.ftype} quant={args.quant}")


if __name__ == "__main__":
    main()

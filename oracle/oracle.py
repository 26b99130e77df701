"""ctypes front-end for the CHECKER libraries (test infrastructure only).

* ``Oracle``  -> oracle/liboracle.so, our C restatement (qmm_oracle.c).
* ``Ref``     -> oracle/_ref/libggml-{base,cpu}.so, the reference's own code compiled by oracle/Makefile
                 from the reference sources (REF_SRC); built where those exist, used as built everywhere else.

oracle/_ref/host holds the reference's host programs (oracle/host.mk) and oracle/_ref/plugin the plugin's objects that
compile against its headers.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
The product (llama.cpp_b200/) must never import it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("LLAMA_CPP_REF", "/root/reference")   # the reference llama.cpp source tree
HOST_DIR = os.path.join(HERE, "_ref", "host")                   # its libllama & co., test-backend-ops, llama-bench, libllama_host.so
PLUGIN_OBJ_DIR = os.path.join(HERE, "_ref", "plugin")

# enum ggml_type values (ggml/include/ggml.h:388-410)
GGML_TYPE_F32, GGML_TYPE_F16 = 0, 1
Q4_0, Q8_0, Q4_K, Q5_K, Q6_K, Q8_K = 2, 8, 12, 13, 14, 15
TYPE_NAMES = {Q4_0: "q4_0", Q8_0: "q8_0", Q4_K: "q4_K", Q5_K: "q5_K", Q6_K: "q6_K"}
BLOCK_ELEMS = {Q4_0: 32, Q8_0: 32, Q4_K: 256, Q5_K: 256, Q6_K: 256, Q8_K: 256}
BLOCK_BYTES = {Q4_0: 18, Q8_0: 34, Q4_K: 144, Q5_K: 176, Q6_K: 210, Q8_K: 292}
ALL_TYPES = (Q4_0, Q8_0, Q4_K, Q5_K, Q6_K)


def row_bytes(t: int, k: int) -> int:
    return k // BLOCK_ELEMS[t] * BLOCK_BYTES[t]


def act_type(t: int) -> int:
    """vec_dot_type of the CPU backend (ggml-cpu/ggml-cpu.c:214-333)."""
    return Q8_K if t in (Q4_K, Q5_K, Q6_K) else Q8_0


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def have_reference() -> bool:
    return os.path.isdir(REF_SRC)


def build(ref: bool = True) -> None:
    """Compile the checker (not the product). The _ref builds need the reference sources; skipped where they are absent."""
    subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])
    if ref and have_reference():
        subprocess.check_call(["make", "-s", "-j8", "-C", HERE, "ref", f"REF={REF_SRC}"])
        subprocess.check_call(["make", "-s", "-j8", "-C", HERE, "-f", "host.mk", "all", f"REF={REF_SRC}"])


class Oracle:
    def __init__(self):
        path = os.path.join(HERE, "liboracle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = self.lib = C.CDLL(path)
        L.orc_fp16_to_fp32.restype = C.c_float
        L.orc_fp16_to_fp32.argtypes = [C.c_uint16]
        L.orc_fp32_to_fp16.restype = C.c_uint16
        L.orc_fp32_to_fp16.argtypes = [C.c_float]
        L.orc_dequantize_row.restype = C.c_int
        L.orc_dequantize_row.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_quantize_row_q8_0.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_quantize_row_q8_K.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_vec_dot.restype = C.c_float
        L.orc_vec_dot.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_void_p]
        L.orc_block_int_dot.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_mul_mat.restype = C.c_int
        L.orc_mul_mat.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64,
                                  C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        L.orc_mul_mat_id.restype = C.c_int
        L.orc_mul_mat_id.argtypes = [C.c_int] + [C.c_int64] * 6 + [C.c_void_p, C.c_int64, C.c_int64,
                                                                    C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]

    def dequantize(self, t: int, blocks: np.ndarray, k: int) -> np.ndarray:
        blocks = np.ascontiguousarray(blocks, dtype=np.uint8)
        out = np.empty(k, dtype=np.float32)
        assert self.lib.orc_dequantize_row(t, _ptr(blocks), _ptr(out), k) == 0
        return out

    def quantize_act(self, t_weight: int, x: np.ndarray) -> np.ndarray:
        """Quantise one f32 row to the activation format the CPU pairs with weight type t_weight."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.size
        at = act_type(t_weight)
        out = np.zeros(row_bytes(at, k), dtype=np.uint8)
        (self.lib.orc_quantize_row_q8_K if at == Q8_K else self.lib.orc_quantize_row_q8_0)(_ptr(x), _ptr(out), k)
        return out

    def vec_dot(self, t: int, k: int, w_row: np.ndarray, act_row: np.ndarray) -> float:
        return float(self.lib.orc_vec_dot(t, k, _ptr(np.ascontiguousarray(w_row)), _ptr(np.ascontiguousarray(act_row))))

    def mul_mat(self, t: int, w: np.ndarray, x: np.ndarray) -> np.ndarray:
        """w: uint8 [M, row_bytes]; x: f32 [N, K] (ggml src1 = [K, N]); returns f32 [N, M] (ggml dst = [M, N])."""
        w = np.ascontiguousarray(w, dtype=np.uint8)
        x = np.ascontiguousarray(x, dtype=np.float32)
        M = w.shape[0]
        N, K = x.shape
        assert w.shape[1] == row_bytes(t, K)
        out = np.empty((N, M), dtype=np.float32)
        rc = self.lib.orc_mul_mat(t, M, N, K, _ptr(w), w.shape[1], _ptr(x), K, _ptr(out), M)
        assert rc == 0, rc
        return out

    def mul_mat_id(self, t: int, w: np.ndarray, b: np.ndarray, ids: np.ndarray) -> np.ndarray:
        """w: uint8 [E, M, row_bytes]; b: f32 [T, nb1, K]; ids: int32 [T, n_used]; returns f32 [T, n_used, M]."""
        w = np.ascontiguousarray(w, dtype=np.uint8)
        b = np.ascontiguousarray(b, dtype=np.float32)
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        E, M, rb = w.shape
        T, nb1, K = b.shape
        n_used = ids.shape[1]
        out = np.empty((T, n_used, M), dtype=np.float32)
        rc = self.lib.orc_mul_mat_id(t, M, K, E, n_used, T, nb1, _ptr(w), rb, M * rb, _ptr(b), _ptr(ids), n_used, _ptr(out))
        assert rc == 0, rc
        return out


class Ref:
    """The reference's own functions (compiled, unmodified, from /root/reference by oracle/Makefile)."""

    def __init__(self):
        d = os.path.join(HERE, "_ref")
        base_p, cpu_p = os.path.join(d, "libggml-base.so"), os.path.join(d, "libggml-cpu.so")
        if not (os.path.exists(base_p) and os.path.exists(cpu_p)):
            raise FileNotFoundError("oracle/_ref not built: run `make -C oracle ref` where /root/reference exists")
        self.base = C.CDLL(base_p, mode=C.RTLD_GLOBAL)
        self.cpu = C.CDLL(cpu_p, mode=C.RTLD_GLOBAL)
        self.cpu.ggml_cpu_init()   # fills ggml_table_f32_f16, which GGML_CPU_FP16_TO_FP32 indexes (simd-mappings.h:144-153)
        b = self.base
        b.ggml_quantize_chunk.restype = C.c_size_t
        b.ggml_quantize_chunk.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]
        b.ggml_fp16_to_fp32.restype = C.c_float
        b.ggml_fp16_to_fp32.argtypes = [C.c_uint16]
        b.ggml_fp32_to_fp16.restype = C.c_uint16
        b.ggml_fp32_to_fp16.argtypes = [C.c_float]
        for n in ("q4_0", "q8_0", "q4_K", "q5_K", "q6_K"):
            getattr(b, f"dequantize_row_{n}").argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        for n in ("quantize_row_q8_0_ref", "quantize_row_q8_K_ref"):
            getattr(b, n).argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        for n in ("quantize_row_q8_0", "quantize_row_q8_K"):
            getattr(self.cpu, n).argtypes = [C.c_void_p, C.c_void_p, C.c_int64]

    def quantize_weights(self, t: int, w: np.ndarray) -> np.ndarray:
        """ggml_quantize_chunk (ggml.c) on f32 [M, K] -> uint8 [M, row_bytes]; what llama-quantize does per tensor."""
        w = np.ascontiguousarray(w, dtype=np.float32)
        M, K = w.shape
        out = np.empty((M, row_bytes(t, K)), dtype=np.uint8)
        n = self.base.ggml_quantize_chunk(t, _ptr(w), _ptr(out), 0, M, K, None)
        assert n == out.size
        return out

    def dequantize(self, t: int, blocks: np.ndarray, k: int) -> np.ndarray:
        blocks = np.ascontiguousarray(blocks, dtype=np.uint8)
        out = np.empty(k, dtype=np.float32)
        getattr(self.base, f"dequantize_row_{TYPE_NAMES[t]}")(_ptr(blocks), _ptr(out), k)
        return out

    def quantize_act(self, t_weight: int, x: np.ndarray, simd: bool = False) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        at = act_type(t_weight)
        out = np.zeros(row_bytes(at, x.size), dtype=np.uint8)
        name = "quantize_row_q8_K" if at == Q8_K else "quantize_row_q8_0"
        fn = getattr(self.cpu, name) if simd else getattr(self.base, name + "_ref")
        fn(_ptr(x), _ptr(out), x.size)
        return out

    def vec_dot(self, t: int, k: int, w_row: np.ndarray, act_row: np.ndarray, generic: bool = True) -> float:
        at = "q8_K" if act_type(t) == Q8_K else "q8_0"
        fn = getattr(self.cpu, f"ggml_vec_dot_{TYPE_NAMES[t]}_{at}" + ("_generic" if generic else ""))
        fn.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
        s = C.c_float(0)
        fn(k, C.byref(s), 0, _ptr(np.ascontiguousarray(w_row)), 0, _ptr(np.ascontiguousarray(act_row)), 0, 1)
        return float(s.value)

    def mul_mat(self, t: int, w: np.ndarray, x: np.ndarray, simd: bool = True) -> np.ndarray:
        """Reference CPU arithmetic for dst = W . X with the reference's OWN compiled kernels (from_float on each
        column, then vec_dot per element), driven over all host threads by oracle.c:orc_mul_mat_with."""
        orc = Oracle().lib
        w = np.ascontiguousarray(w, dtype=np.uint8)
        x = np.ascontiguousarray(x, dtype=np.float32)
        M = w.shape[0]
        N, K = x.shape
        at = act_type(t)
        atn = "q8_K" if at == Q8_K else "q8_0"
        ff = getattr(self.cpu, f"quantize_row_{atn}") if simd else getattr(self.base, f"quantize_row_{atn}_ref")
        vd = getattr(self.cpu, f"ggml_vec_dot_{TYPE_NAMES[t]}_{atn}" + ("" if simd else "_generic"))
        out = np.empty((N, M), dtype=np.float32)
        orc.orc_mul_mat_with.restype = C.c_int
        orc.orc_mul_mat_with.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int64] * 4 + [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        rc = orc.orc_mul_mat_with(C.cast(ff, C.c_void_p), C.cast(vd, C.c_void_p), row_bytes(at, K), M, N, K,
                                  _ptr(w), w.shape[1], _ptr(x), K, _ptr(out), M)
        assert rc == 0
        return out

    # ---- one-node ggml graphs on the reference's CPU backend (ggml_init / ggml_new_tensor_4d / op / ggml_graph_compute_with_ctx)
    def _graph_lib(self):
        b, vp, i64 = self.base, C.c_void_p, C.c_int64
        if getattr(self, "_graph_ready", False):
            return b
        b.ggml_init.restype = vp
        b.ggml_init.argtypes = [_GgmlInitParams]
        b.ggml_free.argtypes = [vp]
        b.ggml_new_tensor_4d.restype = vp
        b.ggml_new_tensor_4d.argtypes = [vp, C.c_int, i64, i64, i64, i64]
        b.ggml_get_data.restype = vp
        b.ggml_get_data.argtypes = [vp]
        b.ggml_nbytes.restype = C.c_size_t
        b.ggml_nbytes.argtypes = [vp]
        b.ggml_flash_attn_ext.restype = vp
        b.ggml_flash_attn_ext.argtypes = [vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float]
        b.ggml_mul_mat_id.restype = vp
        b.ggml_mul_mat_id.argtypes = [vp, vp, vp, vp]
        b.ggml_view_2d.restype = vp
        b.ggml_view_2d.argtypes = [vp, vp, i64, i64, C.c_size_t, C.c_size_t]
        b.ggml_rope_ext.restype = vp
        b.ggml_rope_ext.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int] + [C.c_float] * 6
        b.ggml_new_graph.restype = vp
        b.ggml_new_graph.argtypes = [vp]
        b.ggml_build_forward_expand.argtypes = [vp, vp]
        self.cpu.ggml_graph_compute_with_ctx.restype = C.c_int
        self.cpu.ggml_graph_compute_with_ctx.argtypes = [vp, vp, C.c_int]
        self._graph_ready = True
        return b

    def _run_one_node(self, inputs, make_node, out_shape, mem: int):
        """inputs: list of (ggml type, numpy array in ggml memory order, outermost first[, ggml ne when the array's shape is not it,
        e.g. quantised rows given as bytes]); make_node(ctx, tensors) -> node.  Returns the node's f32 data reshaped to out_shape."""
        b = self._graph_lib()
        ctx = b.ggml_init(_GgmlInitParams(mem + (64 << 20), None, False))
        assert ctx
        try:
            ts = []
            for typ, arr, *given_ne in inputs:
                if arr is None:
                    ts.append(None)
                    continue
                arr = np.ascontiguousarray(arr)
                ne = list(given_ne[0]) + [1] * (4 - len(given_ne[0])) if given_ne else list(arr.shape[::-1]) + [1] * (4 - arr.ndim)
                t = b.ggml_new_tensor_4d(ctx, typ, *ne)
                assert b.ggml_nbytes(t) == arr.nbytes
                C.memmove(b.ggml_get_data(t), arr.ctypes.data, arr.nbytes)
                ts.append(t)
            node = make_node(ctx, ts)
            gf = b.ggml_new_graph(ctx)
            b.ggml_build_forward_expand(gf, node)
            assert self.cpu.ggml_graph_compute_with_ctx(ctx, gf, 4) == 0
            out = np.empty(out_shape, dtype=np.float32)
            assert b.ggml_nbytes(node) == out.nbytes
            C.memmove(out.ctypes.data, b.ggml_get_data(node), out.nbytes)
            return out
        finally:
            b.ggml_free(ctx)

    def flash_attn_ext(self, q, k, v, mask, scale: float, softcap: float = 0.0) -> np.ndarray:
        """ggml_flash_attn_ext on the CPU backend.  Layouts as attention_f64 (q f32 [B, H, N, D], k / v f16 [B, Hkv, n_kv, D],
        mask f16 [m3, m2, >= N, n_kv] or None); returns f32 [B, N, H, DV]."""
        B, H, N, _ = q.shape
        DV = v.shape[3]
        ins = [(GGML_TYPE_F32, q.astype(np.float32)), (GGML_TYPE_F16, k.astype(np.float16)), (GGML_TYPE_F16, v.astype(np.float16)),
               (GGML_TYPE_F16, None if mask is None else mask.astype(np.float16))]
        mem = sum(a.nbytes for _, a in ins if a is not None) + B * N * H * DV * 4
        return self._run_one_node(ins, lambda ctx, t: self.base.ggml_flash_attn_ext(ctx, t[0], t[1], t[2], t[3], scale, 0.0, softcap),
                                  (B, N, H, DV), mem)

    def mul_mat_id(self, t: int, w: np.ndarray, b: np.ndarray, ids: np.ndarray, n_expert_rows: int | None = None) -> np.ndarray:
        """ggml_mul_mat_id on the CPU backend, with the ids built as llama builds them: a ggml_view_2d of the first n_used rows of an
        i32 [n_expert_rows, T] tensor (the top-k argsort), so the view's row stride is n_expert_rows.  Layouts as Oracle.mul_mat_id:
        w uint8 [E, M, row_bytes], b f32 [T, nb1, K], ids int32 [T, n_used]; returns f32 [T, n_used, M]."""
        E, M, rb = w.shape
        T, nb1, K = b.shape
        n_used = ids.shape[1]
        rows = n_expert_rows or E
        full = np.zeros((T, rows), dtype=np.int32)          # the rows past n_used hold ids no view reads
        full[:, :n_used] = ids
        full[:, n_used:] = (np.arange(rows - n_used) % E)[None]
        ins = [(t, np.ascontiguousarray(w, dtype=np.uint8), (K, M, E)), (GGML_TYPE_F32, np.ascontiguousarray(b, dtype=np.float32)), (26, full)]
        mem = w.nbytes + b.nbytes + full.nbytes + T * n_used * M * 4 + (T * nb1 * K * 4 + (64 << 10))
        bl = self._graph_lib()
        return self._run_one_node(ins, lambda ctx, ts: bl.ggml_mul_mat_id(ctx, ts[0], ts[1], bl.ggml_view_2d(ctx, ts[2], n_used, T, rows * 4, 0)),
                                  (T, n_used, M), mem)

    def rope_ext(self, x, pos, n_dims: int, mode: int, freq_base: float = 10000.0, freq_scale: float = 1.0, ext_factor: float = 0.0,
                 attn_factor: float = 1.0, beta_fast: float = 32.0, beta_slow: float = 1.0, n_ctx_orig: int = 0, freq_factors=None) -> np.ndarray:
        """ggml_rope_ext on the CPU backend: x f32 [T, H, D], pos i32 [T], freq_factors f32 [n_dims / 2] or None -> f32 [T, H, D]."""
        x = np.asarray(x, dtype=np.float32)
        ins = [(GGML_TYPE_F32, x), (26, np.asarray(pos, dtype=np.int32)),   # 26 = GGML_TYPE_I32
               (GGML_TYPE_F32, None if freq_factors is None else np.asarray(freq_factors, dtype=np.float32))]
        return self._run_one_node(ins, lambda ctx, t: self.base.ggml_rope_ext(ctx, t[0], t[1], t[2], n_dims, mode, n_ctx_orig, freq_base, freq_scale,
                                                                                ext_factor, attn_factor, beta_fast, beta_slow),
                                  x.shape, 2 * x.nbytes)


_libm = C.CDLL("libm.so.6")
_libm.powf.restype = _libm.logf.restype = C.c_float
_libm.powf.argtypes = [C.c_float, C.c_float]
_libm.logf.argtypes = [C.c_float]
_f32 = np.float32


def attention_f64(q, k, v, mask, scale: float, softcap: float = 0.0, want_abs: bool = False):
    """FLASH_ATTN_EXT (ggml_compute_forward_flash_attn_ext_f16, ggml/src/ggml-cpu/ops.cpp) restated in float64.

    Arrays are in ggml memory order, outermost dimension first: q f32 [B, H, N, DK], k / v f16 [Bk, Hkv, n_kv, D],
    mask f16 [m3, m2, >= N, >= n_kv] or None.  Returns f64 [B, N, H, DV] (ggml dst [DV, H, N, B]) and, with want_abs, also
    A[b, n, h, d] = sum_j p_j |v_jd| / sum_j p_j, the scale a per-element error bound is taken relative to.

    q is rounded to f16 first (K is f16); s = scale * q.k, with softcap: softcap * tanh(s) where scale was divided by softcap
    beforehand (in f32, as ggml does); then + mask.  Keys whose mask is -inf are skipped; a row with no key left gives 0.
    Head h reads kv head h / (H / Hkv), batch b reads b / (B / Bk), the mask plane (h % m2, b % m3)."""
    B, H, N, DK = q.shape
    Bk, Hkv, n_kv, _ = k.shape
    DV = v.shape[3]
    sc = float(_f32(scale) / _f32(softcap)) if softcap != 0.0 else float(scale)
    out = np.zeros((B, N, H, DV))
    A = np.zeros((B, N, H, DV)) if want_abs else None
    q16 = q.astype(np.float16).astype(np.float64)
    g, gb = H // Hkv, B // Bk
    for b in range(B):
        for hk in range(Hkv):
            kk = k[b // gb, hk].astype(np.float64)
            vv = v[b // (B // v.shape[0]), hk].astype(np.float64)
            hs = range(hk * g, (hk + 1) * g)
            s = (q16[b, hk * g:(hk + 1) * g] @ kk.T) * sc
            if softcap != 0.0:
                s = softcap * np.tanh(s)
            if mask is not None:
                m = np.stack([mask[b % mask.shape[0], h % mask.shape[1], :N, :n_kv] for h in hs]).astype(np.float64)
                s = s + m
            live = s != -np.inf
            smax = np.where(live, s, -np.inf).max(-1, keepdims=True)
            p = np.where(live, np.exp(s - np.where(np.isfinite(smax), smax, 0.0)), 0.0)
            l = p.sum(-1, keepdims=True)
            inv = np.where(l > 0, 1.0 / np.where(l > 0, l, 1.0), 0.0)
            out[b, :, hk * g:(hk + 1) * g] = ((p @ vv) * inv).transpose(1, 0, 2)
            if want_abs:
                A[b, :, hk * g:(hk + 1) * g] = ((p @ np.abs(vv)) * inv).transpose(1, 0, 2)
    return (out, A) if want_abs else out


def rope_theta_scale(freq_base: float, n_dims: int) -> np.float32:
    """powf(freq_base, -2.0f / n_dims) with the C library's powf, as ggml computes it on the host."""
    return _f32(_libm.powf(float(freq_base), float(_f32(-2.0) / _f32(n_dims))))


def rope_corr_dims(n_dims: int, n_ctx_orig: int, freq_base: float, beta_fast: float, beta_slow: float):
    """ggml_rope_yarn_corr_dims (ggml/src/ggml.c) in f32."""
    def dim(n_rot):
        num = _f32(_libm.logf(float(_f32(n_ctx_orig) / (_f32(n_rot) * _f32(2) * _f32(np.pi)))))
        return _f32(_f32(n_dims) * num) / _f32(_f32(2) * _f32(_libm.logf(float(freq_base))))
    start, end = np.floor(dim(beta_fast)), np.ceil(dim(beta_slow))
    return _f32(max(0.0, start)), _f32(min(n_dims - 1, end))


def rope_ref(x, pos, n_dims: int, mode: int, freq_base: float = 10000.0, freq_scale: float = 1.0, ext_factor: float = 0.0,
             attn_factor: float = 1.0, beta_fast: float = 32.0, beta_slow: float = 1.0, n_ctx_orig: int = 0, freq_factors=None):
    """ROPE (ggml_compute_forward_rope, modes 0 and 2 = NEOX) of x f32 [T, H, D] (ggml [D, H, T]) at positions pos i32 [T].

    theta is iterated in f32 exactly as ggml_rope_cache_init does (theta *= theta_scale per pair, divided by the pair's
    freq_factor, YaRN ramp and interpolation in f32); cos / sin and the rotation are then taken in float64.  Dims >= n_dims
    pass through.  Returns f64 [T, H, D]."""
    x = np.asarray(x, dtype=np.float32)
    T, H, D = x.shape
    half = n_dims // 2
    ts = rope_theta_scale(freq_base, n_dims)
    corr0, corr1 = rope_corr_dims(n_dims, n_ctx_orig, freq_base, beta_fast, beta_slow)
    fs, ef = _f32(freq_scale), _f32(ext_factor)
    mscale = _f32(attn_factor)
    if ef != 0:
        mscale = _f32(mscale * _f32(_f32(1) + _f32(0.1) * _f32(_libm.logf(float(_f32(1) / fs)))))
    out = x.astype(np.float64).copy()
    for t in range(T):
        theta = _f32(pos[t])
        for i in range(half):
            ff = _f32(freq_factors[i]) if freq_factors is not None else _f32(1)
            th_ex = _f32(theta / ff)
            th_in = _f32(fs * th_ex)
            th = th_in
            if ef != 0:
                y = _f32(_f32(_f32(i) - corr0) /_f32(max(_f32(0.001), _f32(corr1 - corr0))))
                ramp = _f32(_f32(1 - min(_f32(1), max(_f32(0), y))) * ef)
                th = _f32(_f32(th_in * _f32(1 - ramp)) + _f32(th_ex * ramp))
            c, s = np.cos(np.float64(th)) * float(mscale), np.sin(np.float64(th)) * float(mscale)
            ia, ib = (2 * i, 2 * i + 1) if mode == 0 else (i, i + half)
            x0, x1 = x[t, :, ia].astype(np.float64), x[t, :, ib].astype(np.float64)
            out[t, :, ia] = x0 * c - x1 * s
            out[t, :, ib] = x0 * s + x1 * c
            theta = _f32(theta * ts)
    return out


class _GgmlInitParams(C.Structure):
    _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]


def random_blocks(t: int, rows: int, k: int, rng: np.random.Generator, scale: float = 0.02) -> np.ndarray:
    """Random but VALID quantised rows (uint8 [rows, row_bytes]) without running a quantiser:
    random codes/sub-scales, fp16 super-scales sized so dequantised weights are O(scale)."""
    nb = k // BLOCK_ELEMS[t]
    bb = BLOCK_BYTES[t]
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
        q = 15 if t == Q4_K else 31
        put_half(0, u * scale / (32 * q) * 4)
        put_half(2, rng.uniform(0.5, 1.0, size=(rows, nb)) * scale / 32)
    elif t == Q6_K:
        put_half(208, u * scale / (64 * 32) * 2)
    return out.reshape(rows, nb * bb)


def saturated_blocks(t: int, rows: int, k: int, rng: np.random.Generator) -> np.ndarray:
    """K-quant rows whose integer fields are all at their extreme, so that one block's integer sum is as large as the format allows:
    Q4_K / Q5_K every 6-bit scale and min 63 and every quant 15 / 31; Q6_K even rows scale -128 with q = 0 (sc (q - 32) = 4096),
    odd rows scale 127 with q = 63 (3937).  With Q8_K activations of +-127 a block's main sum reaches 256 * 945 * 127 ~ 3.1e7 (Q4_K),
    256 * 1953 * 127 ~ 6.3e7 (Q5_K) and 256 * 4096 * 127 ~ 1.3e8 (Q6_K), all above 2^24.  The fp16 super-scales are random."""
    nb = k // BLOCK_ELEMS[t]
    out = np.zeros((rows, nb, BLOCK_BYTES[t]), dtype=np.uint8)

    def put_half(off, vals):
        h = np.asarray(vals, dtype=np.float16).view(np.uint16)
        out[:, :, off] = (h & 0xFF).astype(np.uint8)
        out[:, :, off + 1] = (h >> 8).astype(np.uint8)

    u = rng.uniform(0.5, 1.0, size=(rows, nb))
    if t in (Q4_K, Q5_K):
        out[:, :, 4:] = 0xFF                                  # scales / mins 63, (Q5_K: qh) and qs: every quant at its maximum
        put_half(0, u * 2.0 ** -12)
        put_half(2, rng.uniform(0.5, 1.0, size=(rows, nb)) * 2.0 ** -12)
    elif t == Q6_K:
        out[1::2, :, :192] = 0xFF                             # odd rows: q = 63 ...
        out[1::2, :, 192:208] = 127                           # ... with scale 127
        out[0::2, :, 192:208] = 0x80                          # even rows: q = 0 with scale -128
        put_half(208, u * 2.0 ** -14)
    else:
        raise ValueError("saturated_blocks: K-quant types only")
    return out.reshape(rows, nb * BLOCK_BYTES[t])


def constant_sign_blocks(n: int, k: int, rng: np.random.Generator) -> np.ndarray:
    """f32 [n, k] activations whose every 256-element block is one value of random sign and size: its Q8_K integers are all +-127."""
    v = rng.uniform(0.25, 2.0, size=(n, k // 256)) * rng.choice([-1.0, 1.0], size=(n, k // 256))
    return np.repeat(v, 256, axis=1).astype(np.float32)

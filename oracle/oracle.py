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

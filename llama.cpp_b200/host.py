"""ctypes binding of include/b200_qmm.h for the Python harness.

torch is used for device memory and streams only; every computation is a call into libb200qmm.so.  If the library
is missing, or there is no sm_90 device, the calls raise -- there is no eager / CPU fallback."""
from __future__ import annotations

import ctypes as C
import os

import torch

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "libb200qmm.so")

Q4_0, Q8_0, Q4_K, Q5_K, Q6_K = 2, 8, 12, 13, 14
BLOCK_ELEMS = {Q4_0: 32, Q8_0: 32, Q4_K: 256, Q5_K: 256, Q6_K: 256}
BLOCK_BYTES = {Q4_0: 18, Q8_0: 34, Q4_K: 144, Q5_K: 176, Q6_K: 210}

_lib = None


class B200Error(RuntimeError):
    pass


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200Error(f"{LIB_PATH} is missing: run llama.cpp_b200/build.py (python -c 'import __graft_entry__ as g; g.build()')")
        L = C.CDLL(LIB_PATH)
        vp, i64, sz, ci = C.c_void_p, C.c_int64, C.c_size_t, C.c_int
        L.b200_qmm_last_error.restype = C.c_char_p
        L.b200_qmm_launch_count.restype = C.c_uint64
        L.b200_row_bytes.restype = i64
        L.b200_row_bytes.argtypes = [ci, i64]
        L.b200_dequantize_rows.argtypes = [ci, vp, i64, vp, i64, i64, i64, vp]
        L.b200_act_workspace_bytes.restype = sz
        L.b200_act_workspace_bytes.argtypes = [ci, i64, i64]
        L.b200_quantize_act.argtypes = [ci, vp, i64, i64, i64, vp, sz, vp]
        L.b200_act_layout.argtypes = [ci, vp, i64, i64] + [C.POINTER(vp)] * 3 + [C.POINTER(i64)] * 3
        L.b200_set_q8_0_rounding.argtypes = [ci]
        L.b200_mul_mat_workspace_bytes.restype = sz
        L.b200_mul_mat_workspace_bytes.argtypes = [ci, i64, i64, i64]
        L.b200_mul_mat.argtypes = [ci, vp, i64, i64, i64, vp, i64, i64, vp, i64, vp, sz, vp]
        L.b200_set_mul_mat_path.argtypes = [ci]
        L.b200_set_gemv_variant.argtypes = [ci]
        L.b200_matvec_program.argtypes = [ci] + [C.c_void_p] * 12 + [C.c_void_p]
        L.b200_matvec_program.restype = ci
        L.b200_gemv_q8.argtypes = [ci, vp, i64, i64, i64, vp, i64, vp, i64, vp]
        L.b200_fused_matvec.argtypes = [ci, ci, vp, vp, vp, i64, vp, vp, C.c_float, ci, vp, vp, vp]
        L.b200_mul_mat_id_workspace_bytes.restype = sz
        L.b200_mul_mat_id_workspace_bytes.argtypes = [ci, i64, i64, i64, i64, i64]
        L.b200_mul_mat_id.argtypes = [ci, vp, i64, i64, i64, i64, i64, vp, i64, vp, i64, i64, i64, vp, vp, sz, vp]
        L.b200_mul_mat_id_path_workspace_bytes.restype = sz
        L.b200_mul_mat_id_path_workspace_bytes.argtypes = [ci, i64, i64, i64, i64, i64, i64]
        L.b200_mul_mat_id_path.argtypes = [ci, vp, i64, i64, i64, i64, i64, vp, i64, vp, i64, i64, i64, vp, vp, sz, ci, C.POINTER(ci), vp]
        L.b200_moe_route_max_tiles.restype = i64
        L.b200_moe_route_max_tiles.argtypes = [i64, i64, i64]
        L.b200_moe_route.restype = i64
        L.b200_moe_route.argtypes = [vp, i64, i64, i64, i64, i64, vp, vp, vp, vp]
        L.b200_mul_mat_host_scratch_bytes.restype = sz
        L.b200_mul_mat_host_scratch_bytes.argtypes = [ci, i64, i64, i64]
        L.b200_mul_mat_host.argtypes = [ci, vp, i64, i64, i64, vp, i64, vp, vp, sz, vp]
        I4 = C.POINTER(i64)
        L.b200_flash_attn_workspace_bytes.restype = sz
        L.b200_flash_attn_workspace_bytes.argtypes = [I4, I4, I4]
        L.b200_flash_attn.argtypes = [vp, I4, I4] * 5 + [C.c_float, C.c_float, vp, sz, ci, vp]
        L.b200_attn_program.argtypes = [C.POINTER(AttnArgs), C.POINTER(ci), vp]
        _lib = L
    return _lib


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise B200Error(f"{what} failed ({rc}): {lib().b200_qmm_last_error().decode()}")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def row_bytes(t: int, k: int) -> int:
    return k // BLOCK_ELEMS[t] * BLOCK_BYTES[t]


def device_count() -> int:
    return int(lib().b200_qmm_device_count())


def launch_count() -> int:
    return int(lib().b200_qmm_launch_count())


def to_device_weights(w_u8) -> torch.Tensor:
    """uint8 [M, row_bytes] (numpy or torch) -> CUDA tensor with 16 bytes of tail slack (ABI contract)."""
    w = torch.as_tensor(w_u8)
    flat = torch.zeros(w.numel() + 16, dtype=torch.uint8, device="cuda")
    flat[: w.numel()] = w.reshape(-1).to("cuda")
    return flat[: w.numel()].view(w.shape)


def dequantize_rows(t: int, w: torch.Tensor, k: int) -> torch.Tensor:
    assert w.is_cuda and w.dtype == torch.uint8 and w.dim() == 2
    y = torch.empty((w.shape[0], k), dtype=torch.float32, device=w.device)
    _check(lib().b200_dequantize_rows(t, w.data_ptr(), w.stride(0), y.data_ptr(), k, w.shape[0], k, _stream()), "b200_dequantize_rows")
    return y


def quantize_act(t_weight: int, x: torch.Tensor):
    """x f32 [N, K] on the GPU -> (qs int8 [N, K], d f32 [N, nd], bsums int16 [N, nb]) as views of one workspace."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    n, k = x.shape
    L = lib()
    nbytes = L.b200_act_workspace_bytes(t_weight, n, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    _check(L.b200_quantize_act(t_weight, x.data_ptr(), x.stride(0), n, k, ws.data_ptr(), nbytes, _stream()), "b200_quantize_act")
    qs, d, bs = C.c_void_p(), C.c_void_p(), C.c_void_p()
    s0, s1, s2 = C.c_int64(), C.c_int64(), C.c_int64()
    _check(L.b200_act_layout(t_weight, ws.data_ptr(), n, k, C.byref(qs), C.byref(d), C.byref(bs), C.byref(s0), C.byref(s1), C.byref(s2)), "b200_act_layout")
    base = ws.data_ptr()

    def view(ptr, dtype, stride, width):
        off = ptr.value - base
        esz = torch.empty(0, dtype=dtype).element_size()
        flat = ws[off: off + n * stride * esz].view(dtype)
        return flat.view(n, stride)[:, :width]

    return view(qs, torch.int8, s0.value, k), view(d, torch.float32, s1.value, s1.value), view(bs, torch.int16, s2.value, s2.value), ws


def mul_mat(t: int, w: torch.Tensor, x: torch.Tensor, out: torch.Tensor | None = None, ws: torch.Tensor | None = None) -> torch.Tensor:
    """w uint8 [M, row_bytes] (rows may be strided), x f32 [N, K] -> f32 [N, M]  (ggml dst = [M, N])."""
    assert w.is_cuda and x.is_cuda and w.dtype == torch.uint8 and x.dtype == torch.float32
    M = w.shape[0]
    N, K = x.shape
    assert w.shape[1] == row_bytes(t, K) and x.stride(1) == 1
    L = lib()
    if out is None:
        out = torch.empty((N, M), dtype=torch.float32, device=x.device)
    need = L.b200_mul_mat_workspace_bytes(t, M, N, K)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=x.device)
    _check(L.b200_mul_mat(t, w.data_ptr(), w.stride(0), M, K, x.data_ptr(), x.stride(0), N, out.data_ptr(), out.stride(0),
                          ws.data_ptr(), ws.numel(), _stream()), "b200_mul_mat")
    return out


def gemv_q8(t: int, w: torch.Tensor, K: int, ws: torch.Tensor, n: int, out: torch.Tensor) -> torch.Tensor:
    """Decode GEMV on activations already quantised into `ws` (quantize_act(...)[3])."""
    _check(lib().b200_gemv_q8(t, w.data_ptr(), w.stride(0), w.shape[0], K, ws.data_ptr(), n, out.data_ptr(), out.stride(0), _stream()), "b200_gemv_q8")
    return out


def fused_matvec(t: int, ws, x: torch.Tensor, norm_w=None, eps: float = 1e-5, mode: int = 0, residual=None, outs=None):
    """The fused decode mat-vec: ws = list of <= 3 uint8 [M_i, row_bytes] weights sharing activation x f32 [K]."""
    n = len(ws)
    K = x.numel()
    if outs is None:
        outs = [torch.empty(w.shape[0], dtype=torch.float32, device=x.device) for w in (ws if mode != 2 else ws[:1])]
    PT = C.c_void_p * 3
    I3 = C.c_int64 * 3
    wp = PT(*[w.data_ptr() for w in ws] + [None] * (3 - n))
    rs = I3(*[w.stride(0) for w in ws] + [0] * (3 - n))
    Ms = I3(*[w.shape[0] for w in ws] + [0] * (3 - n))
    dp = PT(*([o.data_ptr() for o in outs] + [None] * (3 - len(outs))))
    rp = PT(*([r.data_ptr() for r in residual] + [None] * (3 - len(residual)))) if residual else None
    _check(lib().b200_fused_matvec(t, n, wp, rs, Ms, K, x.data_ptr(), norm_w.data_ptr() if norm_w is not None else None, eps, mode,
                                   rp, dp, _stream()), "b200_fused_matvec")
    return outs


def matvec_program(phases):
    """phases: list of dicts {type, ws:[<=3 weights], x, norm_w|None, eps, mode, residual|None, outs:[tensors]} run as ONE
    persistent-kernel launch (b200_matvec_program)."""
    n = len(phases)
    IA, I64, PT, FA = C.c_int * n, C.c_int64 * n, C.c_void_p * n, C.c_float * n
    P3, I3 = C.c_void_p * (3 * n), C.c_int64 * (3 * n)
    w3, rs3, m3, d3, t3 = [None] * (3 * n), [0] * (3 * n), [0] * (3 * n), [None] * (3 * n), [0] * (3 * n)
    for i, p in enumerate(phases):
        for j, w in enumerate(p["ws"]):
            w3[3 * i + j] = w.data_ptr(); rs3[3 * i + j] = w.stride(0); m3[3 * i + j] = w.shape[0]
            t3[3 * i + j] = p["types"][j] if "types" in p else p["type"]
        for j, o in enumerate(p["outs"]):
            d3[3 * i + j] = o.data_ptr()
        if p.get("mode", 0) == 2:
            d3[3 * i + 1] = d3[3 * i]
    _check(lib().b200_matvec_program(
        n, (C.c_int * (3 * n))(*t3), IA(*[len(p["ws"]) for p in phases]), P3(*w3), I3(*rs3), I3(*m3),
        I64(*[p["x"].numel() for p in phases]), PT(*[p["x"].data_ptr() for p in phases]),
        PT(*[p["norm_w"].data_ptr() if p.get("norm_w") is not None else None for p in phases]), FA(*[p.get("eps", 1e-5) for p in phases]),
        IA(*[p.get("mode", 0) for p in phases]), PT(*[p["residual"].data_ptr() if p.get("residual") is not None else None for p in phases]),
        P3(*d3), _stream()), "b200_matvec_program")


def _ggml_view(t: torch.Tensor | None):
    """A torch tensor (any strides, <= 4 dims, outermost first) as ggml's (data, ne[4], nb[4] in bytes)."""
    if t is None:
        return None, None, None
    assert t.dim() <= 4
    shape = [1] * (4 - t.dim()) + list(t.shape)
    stride = [0] * (4 - t.dim()) + list(t.stride())
    ne = (C.c_int64 * 4)(*shape[::-1])
    nb = (C.c_int64 * 4)(*[s * t.element_size() for s in stride[::-1]])
    return t.data_ptr(), ne, nb


def flash_attn_workspace_bytes(q: torch.Tensor, k: torch.Tensor, mask: torch.Tensor | None) -> int:
    return int(lib().b200_flash_attn_workspace_bytes(_ggml_view(q)[1], _ggml_view(k)[1], _ggml_view(mask)[1]))


def flash_attn(q, k, v, mask, dst, scale: float, softcap: float = 0.0, ws: torch.Tensor | None = None, path: int = 0) -> torch.Tensor:
    """FLASH_ATTN_EXT (b200_flash_attn).  Tensors outermost dimension first, ggml's order reversed: q f32 [B, H, N, D], k / v f16
    [Bk, Hkv, n_kv, D], mask f16 [m3, m2, >= N, >= n_kv] or None, dst f32 [B, N, H, DV]; any strides (views of a cache,
    llama's permuted q).  path 0 auto, 1 scalar kernel, 2 tensor-core kernel; ws: scratch for the tile pre-pass or None."""
    args = []
    for t in (q, k, v, mask, dst):
        args += list(_ggml_view(t))
    _check(lib().b200_flash_attn(*args, scale, softcap, ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0, path,
                                 _stream()), "b200_flash_attn")
    return dst


class AttnArgs(C.Structure):
    """include/b200_qmm.h: b200_attn_args."""
    _fields_ = [("type_qkv", C.c_int * 3), ("w_qkv", C.c_void_p * 3), ("row_stride_qkv", C.c_int64 * 3),
                ("x", C.c_void_p), ("norm_w", C.c_void_p), ("n_embd", C.c_int64), ("eps", C.c_float),
                ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p),
                ("n_head", C.c_int), ("n_head_kv", C.c_int), ("head_dim", C.c_int), ("n_dims", C.c_int), ("rope_mode", C.c_int), ("n_ctx_orig", C.c_int),
                ("freq_base", C.c_float), ("freq_scale", C.c_float), ("ext_factor", C.c_float), ("attn_factor", C.c_float),
                ("beta_fast", C.c_float), ("beta_slow", C.c_float),
                ("freq_factors", C.c_void_p), ("pos", C.c_void_p),
                ("k_cache", C.c_void_p), ("k_row_bytes", C.c_int64), ("v_cache", C.c_void_p), ("v_row_bytes", C.c_int64),
                ("kpos", C.c_void_p), ("vpos", C.c_void_p),
                ("kview", C.c_void_p), ("k_nb1", C.c_int64), ("k_nb2", C.c_int64),
                ("vview", C.c_void_p), ("v_nb1", C.c_int64), ("v_nb2", C.c_int64), ("n_kv", C.c_int),
                ("mask", C.c_void_p), ("scale", C.c_float), ("softcap", C.c_float), ("dst", C.c_void_p)]


def attn_program(q, k, v, dst, k_cache, v_cache, kpos, vpos, pos, n_head: int, n_head_kv: int, n_kv: int, scale: float, softcap: float = 0.0,
                 mask=None, n_dims: int = 128, rope_mode: int = 0, freq_base: float = 10000.0, freq_scale: float = 1.0, ext_factor: float = 0.0,
                 attn_factor: float = 1.0, beta_fast: float = 32.0, beta_slow: float = 1.0, n_ctx_orig: int = 0, freq_factors=None,
                 qkv=None) -> int:
    """One persistent-kernel launch of the decode attention phase (b200_attn_program); returns the planned nsplit.
    k_cache / v_cache f16 [n_cells, n_head_kv, 128] (the K / V views are their first n_kv cells); kpos / vpos i64 [1], pos i32 [1]
    on the device; mask f16 [n_kv] or None.  qkv = dict(types, ws:[3 weights], x, norm_w, eps) runs the q|k|v mat-vec in the
    same launch, writing q, k, v as well."""
    a = AttnArgs()
    D = k_cache.shape[-1]
    if qkv is not None:
        for j in range(3):
            a.type_qkv[j] = qkv["types"][j]; a.w_qkv[j] = qkv["ws"][j].data_ptr(); a.row_stride_qkv[j] = qkv["ws"][j].stride(0)
        a.x = qkv["x"].data_ptr(); a.n_embd = qkv["x"].numel(); a.eps = qkv.get("eps", 1e-5)
        a.norm_w = qkv["norm_w"].data_ptr() if qkv.get("norm_w") is not None else None
    a.q, a.k, a.v, a.dst = q.data_ptr(), k.data_ptr(), v.data_ptr(), dst.data_ptr()
    a.n_head, a.n_head_kv, a.head_dim, a.n_dims, a.rope_mode, a.n_ctx_orig = n_head, n_head_kv, D, n_dims, rope_mode, n_ctx_orig
    a.freq_base, a.freq_scale, a.ext_factor, a.attn_factor, a.beta_fast, a.beta_slow = freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow
    a.freq_factors = freq_factors.data_ptr() if freq_factors is not None else None
    a.pos = pos.data_ptr()
    a.k_cache, a.k_row_bytes = k_cache.data_ptr(), k_cache.stride(0) * 2
    a.v_cache, a.v_row_bytes = v_cache.data_ptr(), v_cache.stride(0) * 2
    a.kpos, a.vpos = kpos.data_ptr(), vpos.data_ptr()
    a.kview, a.k_nb1, a.k_nb2 = k_cache.data_ptr(), k_cache.stride(0) * 2, k_cache.stride(1) * 2
    a.vview, a.v_nb1, a.v_nb2 = v_cache.data_ptr(), v_cache.stride(0) * 2, v_cache.stride(1) * 2
    a.n_kv = n_kv
    a.mask = mask.data_ptr() if mask is not None else None
    a.scale, a.softcap = scale, softcap
    ns = C.c_int(0)
    _check(lib().b200_attn_program(C.byref(a), C.byref(ns), _stream()), "b200_attn_program")
    return ns.value


def mul_mat_id(t: int, w: torch.Tensor, b: torch.Tensor, ids: torch.Tensor, path: int | None = None, out: torch.Tensor | None = None):
    """w uint8 [E, M, row_bytes]; b f32 [T, nb1, K]; ids int32 [T, n_used] (any row stride, e.g. the first n_used columns of an
    [T, n_expert] argsort) -> f32 [T, n_used, M].
    path None: b200_mul_mat_id (the routed GEMV), returns out.  path 0 / 1 / 2: b200_mul_mat_id_path (0 the backend's choice, 1 the
    routed GEMV, 2 the grouped GEMM), returns (out, the kernel taken: 1 GEMV, 2 grouped GEMM).  out: the dst tensor to write."""
    E, M, rb = w.shape
    T, nb1, K = b.shape
    n_used = ids.shape[1]
    assert b.is_contiguous() and ids.dtype == torch.int32 and ids.stride(1) == 1
    L = lib()
    if out is None:
        out = torch.empty((T, n_used, M), dtype=torch.float32, device=b.device)
    assert out.shape == (T, n_used, M) and out.is_contiguous()
    if path is None:
        need = L.b200_mul_mat_id_workspace_bytes(t, M, K, n_used, T, nb1)
        ws = torch.empty(need, dtype=torch.uint8, device=b.device)
        _check(L.b200_mul_mat_id(t, w.data_ptr(), w.stride(1), w.stride(0), E, M, K, b.data_ptr(), nb1, ids.data_ptr(), ids.stride(0),
                                 n_used, T, out.data_ptr(), ws.data_ptr(), need, _stream()), "b200_mul_mat_id")
        return out
    need = L.b200_mul_mat_id_path_workspace_bytes(t, M, K, E, n_used, T, nb1)
    ws = torch.empty(need, dtype=torch.uint8, device=b.device)
    taken = C.c_int(0)
    _check(L.b200_mul_mat_id_path(t, w.data_ptr(), w.stride(1), w.stride(0), E, M, K, b.data_ptr(), nb1, ids.data_ptr(), ids.stride(0),
                                  n_used, T, out.data_ptr(), ws.data_ptr(), need, path, C.byref(taken), _stream()), "b200_mul_mat_id_path")
    return out, taken.value


def moe_route(ids: torch.Tensor, n_expert: int, nb1: int):
    """The grouped GEMM's router alone (b200_moe_route): ids int32 [T, n_used] (any row stride) -> (tile_expert int32 [max_tiles],
    col_src int32 [max_tiles, 128], col_dst int32 [max_tiles, 128])."""
    T, n_used = ids.shape
    assert ids.is_cuda and ids.dtype == torch.int32 and ids.stride(1) == 1
    L = lib()
    mt = int(L.b200_moe_route_max_tiles(n_expert, n_used, T))
    te = torch.empty(mt, dtype=torch.int32, device=ids.device)
    cs = torch.empty((mt, 128), dtype=torch.int32, device=ids.device)
    cd = torch.empty((mt, 128), dtype=torch.int32, device=ids.device)
    rc = L.b200_moe_route(ids.data_ptr(), ids.stride(0), n_expert, n_used, T, nb1, te.data_ptr(), cs.data_ptr(), cd.data_ptr(), _stream())
    _check(0 if rc >= 0 else rc, "b200_moe_route")
    assert rc == mt
    return te, cs, cd


class HostMulMat:
    """End-to-end call with HOST buffers (pinned): the `e2e` leg of bench.py.  Weights stay resident in HBM."""

    def __init__(self, t: int, w: torch.Tensor, N: int, K: int):
        self.t, self.w, self.N, self.K, self.M = t, w, N, K, w.shape[0]
        n = lib().b200_mul_mat_host_scratch_bytes(t, self.M, N, K)
        self.scratch = torch.empty(n, dtype=torch.uint8, device=w.device)
        self.x_host = torch.empty((N, K), dtype=torch.float32).pin_memory()
        self.y_host = torch.empty((N, self.M), dtype=torch.float32).pin_memory()

    def __call__(self) -> torch.Tensor:
        _check(lib().b200_mul_mat_host(self.t, self.w.data_ptr(), self.w.stride(0), self.M, self.K, self.x_host.data_ptr(), self.N,
                                       self.y_host.data_ptr(), self.scratch.data_ptr(), self.scratch.numel(), _stream()), "b200_mul_mat_host")
        return self.y_host

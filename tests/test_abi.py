"""CPU-only: the C-ABI library builds, loads, and exports every symbol include/b200_qmm.h declares; argument checks
that need no GPU behave; the product never imports the oracle."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "llama.cpp_b200", "libb200qmm.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        subprocess.check_call(["make", "-s", "-j8", "-C", os.path.join(ROOT, "llama.cpp_b200", "csrc")])
    return C.CDLL(LIB)


def declared_symbols(header):
    txt = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", txt)))


def test_every_declared_symbol_is_exported(lib):
    syms = declared_symbols("b200_qmm.h")
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b200_qmm.h but not exported by libb200qmm.so"


def test_every_attention_symbol_is_exported(lib):
    syms = declared_symbols("b200_attn.h")
    assert syms == ["b200_attn_program", "b200_flash_attn", "b200_flash_attn_workspace_bytes"]
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b200_attn.h but not exported by libb200qmm.so"


def test_every_moe_symbol_is_exported(lib):
    syms = declared_symbols("b200_moe.h")
    assert syms == ["b200_moe_route", "b200_moe_route_max_tiles", "b200_mul_mat_id_path", "b200_mul_mat_id_path_workspace_bytes"]
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b200_moe.h but not exported by libb200qmm.so"


def test_plugin_exports_every_symbol_its_header_declares():
    """libggml-b200.so (the drop-in boundary): the two dl entry points + the bench hooks of include/ggml-b200.h, and the
    kernel C ABI it embeds.  Symbol table only -- loading it needs libggml-base and calling it needs a GPU."""
    plugin = os.path.join(ROOT, "llama.cpp_b200", "libggml-b200.so")
    if not os.path.exists(plugin):
        pytest.skip("plugin not built (its C++ objects need the reference's headers)")
    out = subprocess.check_output(["nm", "-D", "--defined-only", plugin], text=True)
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    txt = open(os.path.join(ROOT, "include", "ggml-b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)   # declarations only, not the prose
    declared = set(re.findall(r"\b(ggml_b(?:ackend|200)_[a-z0-9_]+)\s*\(", txt))
    assert {"ggml_backend_init", "ggml_backend_score"} <= declared
    for s in sorted(declared):
        assert s in exported, f"{s} declared in include/ggml-b200.h but not exported by libggml-b200.so"
    for s in declared_symbols("b200_qmm.h") + declared_symbols("b200_attn.h") + declared_symbols("b200_moe.h"):
        assert s in exported, s


def test_abi_version_and_row_bytes(lib):
    assert lib.b200_qmm_abi_version() == 1
    lib.b200_row_bytes.restype = C.c_int64
    lib.b200_row_bytes.argtypes = [C.c_int, C.c_int64]
    assert lib.b200_row_bytes(12, 4096) == 2304      # Q4_K
    assert lib.b200_row_bytes(14, 14336) == 11760    # Q6_K
    assert lib.b200_row_bytes(2, 2880) == 1620       # Q4_0, rows not 16-byte multiples
    assert lib.b200_row_bytes(12, 100) == 0          # ragged K rejected
    assert lib.b200_row_bytes(99, 256) == 0          # unknown type


def test_bad_arguments_fail_before_touching_the_gpu(lib):
    lib.b200_qmm_last_error.restype = C.c_char_p
    lib.b200_mul_mat.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                 C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]
    assert lib.b200_mul_mat(12, None, 0, 16, 100, None, 0, 1, None, 0, None, 0, None) == -1     # K % 256 != 0
    assert b"bad type/shape" in lib.b200_qmm_last_error()
    assert lib.b200_mul_mat(12, None, 0, 16, 256, None, 0, 1, None, 0, None, 0, None) == -3     # workspace too small
    assert lib.b200_mul_mat(12, None, 0, 0, 256, None, 0, 1, None, 0, None, 1 << 20, None) == 0  # empty M is a no-op


def test_no_gpu_means_no_devices_not_a_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.b200_qmm_device_count() == 0


def test_product_never_references_the_oracle():
    """No source of the product, of the host driver, of bench data generation names the checker; and the built shared objects
    neither need nor search it (DT_NEEDED / RPATH / RUNPATH and every string of the binaries)."""
    srcs = []
    for top in ("llama.cpp_b200", "host", "tools", "include"):
        for d, dirs, files in os.walk(os.path.join(ROOT, top)):
            dirs[:] = [x for x in dirs if x not in ("_ref", "__pycache__")]
            srcs += [os.path.join(d, f) for f in files if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", "Makefile"))]
    # tools that exist to DIAGNOSE against the checker are test infrastructure, not product
    srcs = [f for f in srcs if os.path.basename(f) not in ("diag_logits.py", "diag_mega.py", "diag_race.py", "gemv_sweep.py", "gemm_sweep.py", "ncu_one_gemm.py")]
    assert len(srcs) > 20
    for f in srcs:
        txt = open(f, errors="ignore").read()
        for needle in ("liboracle", "qmm_oracle", "from oracle", "import oracle", "oracle/_ref", "../oracle", "oracle.oracle"):
            assert needle not in txt, (f, needle)
    for so in ("llama.cpp_b200/libb200qmm.so", "llama.cpp_b200/libggml-b200.so", "oracle/_ref/host/libllama_host.so"):
        path = os.path.join(ROOT, so)
        if not os.path.exists(path):
            continue
        dyn = subprocess.check_output(["readelf", "-d", path], text=True)
        assert "oracle" not in dyn, (so, dyn)
        assert b"oracle" not in open(path, "rb").read(), so


def test_sass_has_no_local_memory_in_gemv():
    log = os.path.join(ROOT, "llama.cpp_b200", "csrc", "gemv.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("no ptxas log")
    txt = open(log).read()
    # batch-1 instantiations (NCOLS = 1) are the decode hot path: they must not spill
    entries = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", txt)
    hot = [e for e in entries if re.search(r"gemv_q_kernelILi\d+ELi1EE", e[0])]
    assert len(hot) == 5
    for name, stack, st, ld in hot:
        assert int(st) == 0 and int(ld) == 0 and int(stack) == 0, (name, stack, st, ld)


def test_attention_arguments_fail_before_touching_the_gpu(lib):
    """b200_flash_attn / b200_attn_program reject unsupported or inconsistent shapes on the host (no device memory is named)."""
    lib.b200_qmm_last_error.restype = C.c_char_p
    I4 = C.c_int64 * 4
    vp = C.c_void_p
    lib.b200_flash_attn.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)] * 5 + [C.c_float, C.c_float, vp, C.c_size_t, C.c_int, vp]

    def fa(D, N, H, Hkv, path, n_kv=64):
        q_ne, k_ne, d_ne = I4(D, N, H, 1), I4(D, n_kv, Hkv, 1), I4(D, H, N, 1)
        q_nb, k_nb, d_nb = I4(4, 4 * D, 4 * D * N, 4 * D * N * H), I4(2, 2 * D, 2 * D * n_kv, 2 * D * n_kv * Hkv), I4(4, 4 * D, 4 * D * H, 4 * D * H * N)
        return lib.b200_flash_attn(None, q_ne, q_nb, None, k_ne, k_nb, None, k_ne, k_nb, None, None, None, None, d_ne, d_nb,
                                   0.1, 0.0, None, 0, path, None)

    assert fa(96, 32, 4, 4, 2) == -6                         # the tensor-core kernel: D in {64, 128} only, no fall-back
    assert b"tensor-core" in lib.b200_qmm_last_error()
    assert fa(256, 32, 4, 4, 2) == -6
    assert fa(128, 15, 4, 4, 2) == -6                        # ... and >= 16 rows
    assert fa(320, 1, 4, 4, 1) == -6                         # the scalar kernel: D <= 256
    assert fa(128, 4, 6, 4, 1) == -1                         # H not a multiple of Hkv
    assert fa(128, 4, 4, 4, 3) == -1                         # unknown path

    class Args(C.Structure):                                  # the leading fields of b200_attn_args, the rest zero
        _fields_ = [("type_qkv", C.c_int * 3), ("w_qkv", vp * 3), ("row_stride_qkv", C.c_int64 * 3), ("x", vp), ("norm_w", vp),
                    ("n_embd", C.c_int64), ("eps", C.c_float), ("q", vp), ("k", vp), ("v", vp),
                    ("n_head", C.c_int), ("n_head_kv", C.c_int), ("head_dim", C.c_int), ("n_dims", C.c_int), ("rope_mode", C.c_int),
                    ("pad", C.c_char * 512)]

    lib.b200_attn_program.argtypes = [C.POINTER(Args), C.POINTER(C.c_int), vp]
    a = Args(n_head=32, n_head_kv=8, head_dim=64, n_dims=64)
    assert lib.b200_attn_program(C.byref(a), None, None) == -6   # head_dim != 128
    assert b"head_dim" in lib.b200_qmm_last_error()
    a = Args(n_head=32, n_head_kv=6, head_dim=128, n_dims=128)
    assert lib.b200_attn_program(C.byref(a), None, None) == -1   # n_head not a multiple of n_head_kv
    assert b"n_head_kv" in lib.b200_qmm_last_error()
    assert lib.b200_attn_program(None, None, None) == -1


def test_moe_arguments_fail_before_touching_the_gpu(lib):
    """b200_mul_mat_id_path / b200_moe_route reject a bad path, nb1 or n_used on the host (no device memory is named)."""
    lib.b200_qmm_last_error.restype = C.c_char_p
    vp, i64 = C.c_void_p, C.c_int64
    lib.b200_mul_mat_id_path.argtypes = [C.c_int, vp, i64, i64, i64, i64, i64, vp, i64, vp, i64, i64, i64, vp, vp, C.c_size_t, C.c_int,
                                         C.POINTER(C.c_int), vp]
    lib.b200_moe_route.restype = i64
    lib.b200_moe_route.argtypes = [vp, i64, i64, i64, i64, i64, vp, vp, vp, vp]
    lib.b200_moe_route_max_tiles.restype = i64
    lib.b200_moe_route_max_tiles.argtypes = [i64, i64, i64]
    taken = C.c_int(7)

    def mmid(path, nb1=2, n_used=2, t=12, E=8, T=16, ws=1 << 30):
        return lib.b200_mul_mat_id_path(t, None, 144, 144 * 64, E, 64, 256, None, nb1, None, E, n_used, T, None, None, ws, path,
                                        C.byref(taken), None)

    assert mmid(3) == -1 and b"path" in lib.b200_qmm_last_error()
    assert taken.value == 0                                   # nothing ran
    assert mmid(-1) == -1
    assert mmid(0, nb1=3) == -1 and b"nb1" in lib.b200_qmm_last_error()
    assert mmid(1, nb1=2, n_used=4) == -1
    assert mmid(2, n_used=0, nb1=1) == -1 and b"n_used" in lib.b200_qmm_last_error()
    assert mmid(1, n_used=-2, nb1=1) == -1
    assert mmid(0, t=99) == -1                                # unknown type
    assert mmid(2, ws=0) == -3                                # workspace too small
    assert mmid(2, T=0) == 0                                  # no tokens: a no-op
    assert lib.b200_moe_route_max_tiles(8, 2, 100) == 2 + 8   # ceil(200 / 128) + n_expert
    assert lib.b200_moe_route_max_tiles(60, 4, 32) == 1 + 60
    assert lib.b200_moe_route(C.c_void_p(16), 8, 8, 2, 4, 3, C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), None) == -1   # nb1
    assert lib.b200_moe_route(C.c_void_p(16), 8, 8, 0, 4, 1, C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), None) == -1   # n_used
    assert lib.b200_moe_route(C.c_void_p(16), 257, 257, 2, 4, 1, C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), None) == -6
    assert b"256" in lib.b200_qmm_last_error()

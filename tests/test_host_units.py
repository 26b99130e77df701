"""CPU-only: the kernels' index math (qmm_formats.cuh), compiled for the host, against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle.oracle import ALL_TYPES, Q8_K, act_type, random_blocks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hu():
    so = os.path.join(ROOT, "tests", "_host_units.so")
    src = os.path.join(ROOT, "tests", "host_units.cpp")
    hdr = os.path.join(ROOT, "llama.cpp_b200", "csrc", "qmm_formats.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-x", "c++", src, "-o", so])
    lib = C.CDLL(so)
    lib.hu_row_dot.restype = C.c_float
    lib.hu_row_dot.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4
    lib.hu_dequant_row.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    return lib


def act_soa(t, blocks, k):
    """ggml block_q8_K / block_q8_0 bytes -> our ActQ8 planes (qs, d, bsums)."""
    if act_type(t) == Q8_K:
        b = blocks.reshape(k // 256, 292)
        d = b[:, :4].copy().view(np.float32).reshape(-1)
        qs = b[:, 4:260].copy().view(np.int8).reshape(-1)
        bs = b[:, 260:].copy().view(np.int16).reshape(-1)
    else:
        b = blocks.reshape(k // 32, 34)
        d = b[:, :2].copy().view(np.float16).astype(np.float32).reshape(-1)
        qs = b[:, 2:].copy().view(np.int8).reshape(-1)
        bs = qs.reshape(-1, 32).astype(np.int32).sum(axis=1).astype(np.int16)
    return np.ascontiguousarray(qs), np.ascontiguousarray(d), np.ascontiguousarray(bs)


@pytest.mark.parametrize("t", ALL_TYPES)
@pytest.mark.parametrize("K", [256, 2048, 2304, 4096, 4352])
def test_row_dot_matches_oracle(hu, oracle, t, K):
    rng = np.random.default_rng(K + t)
    w = random_blocks(t, 3, K, rng)
    x = rng.standard_normal(K).astype(np.float32)
    a = oracle.quantize_act(t, x)
    qs, d, bs = act_soa(t, a, K)
    for m in range(3):
        wr = np.concatenate([w[m], np.zeros(32, np.uint8)])   # read slack, as the staging ring provides
        got = hu.hu_row_dot(t, K, wr.ctypes.data, qs.ctypes.data, d.ctypes.data, bs.ctypes.data)
        want = oracle.vec_dot(t, K, w[m], a)
        scale = float(np.abs(oracle.dequantize(t, w[m], K) * x).sum())
        assert abs(got - want) <= 3e-6 * scale, (t, K, m, got, want)


@pytest.mark.parametrize("t", ALL_TYPES)
def test_dequant_elem_bit_exact(hu, oracle, t):
    rng = np.random.default_rng(t)
    K = 1024
    w = random_blocks(t, 4, K, rng)
    for m in range(4):
        y = np.empty(K, np.float32)
        hu.hu_dequant_row(t, w[m].ctypes.data, y.ctypes.data, K)
        assert np.array_equal(y.view(np.uint32), oracle.dequantize(t, w[m], K).view(np.uint32))


def test_gemm_prepass_chunk_layout(hu):
    """The warp-per-block activation pre-pass stores one 16-byte chunk per lane; its element order and address must equal the
    per-element swizzled K-major addressing (gemm_layout.cuh) that the weight de-quantiser and the wgmma descriptors assume."""
    assert hu.hu_prepass_layout_mismatches(128) == 0

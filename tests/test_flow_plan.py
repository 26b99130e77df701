"""CPU-only: the host-side work plan of the persistent dataflow decode kernel (csrc/decode_flow.cu, FlowBuilder::add_matvec).
For every mat-vec shape of the models BASELINE.json names, the plan must cut the rows into ring pieces that fit a slot, that one
producer warp can issue (<= 32 bulk copies), and whose lanes cover every 256-weight block of a row exactly once."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "llama.cpp_b200", "libb200qmm.so")
Q4_K, Q5_K, Q6_K = 12, 13, 14
BB = {Q4_K: 144, Q5_K: 176, Q6_K: 210}


def plan(types, Ms, K, mode=0, norm=False, grid=132, strides=None):
    L = C.CDLL(LIB)
    L.b200_flow_plan.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    n = len(types)
    rs = strides or [K // 256 * BB.get(t, 144) for t in types]
    out = (C.c_int * 8)()
    rc = L.b200_flow_plan(n, (C.c_int * n)(*types), (C.c_int64 * n)(*Ms), K, (C.c_int64 * n)(*rs), mode, int(norm), grid, out)
    return rc, list(out)


SHAPES = [
    # (types, Ms, K, mode, norm)                                                  Llama-3-8B Q4_K_M
    ([Q4_K, Q4_K, Q6_K], [4096, 1024, 1024], 4096, 0, True), ([Q4_K, Q4_K, Q4_K], [4096, 1024, 1024], 4096, 0, True),
    ([Q4_K], [4096], 4096, 1, False), ([Q4_K, Q4_K], [14336, 14336], 4096, 2, True),
    ([Q4_K], [4096], 14336, 1, False), ([Q6_K], [4096], 14336, 1, False), ([Q6_K], [128256], 4096, 0, True),
    # Llama-3-70B, one GPU's share under -sm tensor x8 and the full matrices
    ([Q4_K, Q4_K, Q5_K], [1024, 128, 128], 8192, 0, True), ([Q4_K], [8192], 1024, 1, False), ([Q4_K, Q4_K], [3584, 3584], 8192, 2, True),
    ([Q6_K], [8192], 3584, 1, False), ([Q4_K, Q4_K], [28672, 28672], 8192, 2, True),
    # Q5_K_M mixes, the tiny/small test presets
    ([Q5_K, Q5_K, Q6_K], [4096, 1024, 1024], 4096, 0, True), ([Q5_K], [1024], 2816, 1, False), ([Q4_K, Q4_K, Q6_K], [256, 128, 128], 256, 0, True),
    ([Q6_K], [512], 256, 0, True), ([Q4_K], [4096], 11008, 1, False),
]
# Llama-3-8B under -sm tensor x2 / x4 / x8 (what bench.py --gpus N hands every GPU): column-parallel q|k|v and gate|up keep K and shrink M,
# row-parallel attn_output and ffn_down shrink K (512 .. 2048, 1792 .. 7168); in the meta backend's node order q is its own phase and v|k share one
for tp in (2, 4, 8):
    SHAPES += [([Q4_K], [4096 // tp], 4096, 0, True), ([Q6_K, Q4_K], [1024 // tp, 1024 // tp], 4096, 0, True),
               ([Q4_K], [4096], 4096 // tp, 0, False), ([Q4_K, Q4_K], [14336 // tp, 14336 // tp], 4096, 2, True),
               ([Q6_K], [4096], 14336 // tp, 0, False), ([Q4_K], [4096], 14336 // tp, 0, False), ([Q6_K], [128256 // tp], 4096, 0, True)]


@pytest.mark.parametrize("types,Ms,K,mode,norm", SHAPES)
def test_plan_fits_the_ring(types, Ms, K, mode, norm):
    if not os.path.exists(LIB):
        pytest.skip("libb200qmm.so not built")
    rc, (S, seg, RP, R0, R1, R2, keep_h, slot) = plan(types, Ms, K, mode, norm)
    assert rc == 0
    nblk = K // 256
    assert S in (1, 2) and S * seg >= nblk and (S - 1) * seg < nblk          # the segments tile the row
    assert seg <= 32 and RP * seg <= 32 and RP >= 1                           # one lane per block of a warp step
    if RP > 1:
        assert seg & (seg - 1) == 0                                           # aligned power-of-two lane groups for the row reduction
    sub = 2 if mode == 2 else 1
    for t, R in zip(types, (R0, R1, R2)):
        assert R >= 1
        row_bytes = nblk * BB[t]
        if S == 1:                                                            # dense rows: one copy per sub-piece
            assert sub * ((R * row_bytes + 16 + 15) // 16 * 16) <= slot
        else:                                                                 # one copy per (sub-piece, row)
            assert sub * R <= 32 and sub * R * ((seg * BB[t] + 16 + 15) // 16 * 16) <= slot
    assert keep_h == (1 if norm and K <= 8192 else 0)


def test_unsupported_shapes_are_declined_not_mangled():
    if not os.path.exists(LIB):
        pytest.skip("libb200qmm.so not built")
    assert plan([Q4_K], [4096], 28672)[0] != 0            # K > 16384: more activation blocks than the kernel holds
    assert plan([Q4_K], [4096], 4000)[0] != 0             # ragged K
    assert plan([Q4_K, Q4_K], [64, 64], 14336)[0] != 0    # split rows: single matrix only
    assert plan([2], [4096], 4096)[0] != 0                # Q4_0 is not a K-quant
    assert plan([Q4_K], [4096], 8192 + 256, norm=True)[0] != 0   # a fused RMS_NORM needs the vector in one prologue pass


def test_postponed_rope_names_the_remembered_q_vector():
    """The meta backend's node order (-sm tensor): q mat-vec, ROPE(q) postponed, v | k mat-vecs whose outputs may reuse the q mat-mul's
    buffer, then the attention phase.  The recorder looks vectors up by address; the attention phase must use the q vector remembered at
    the postponement (the round-2 tensor-parallel failure: it read v's slots as q).  Host-only check through the C ABI."""
    L = C.CDLL(os.path.join(ROOT, "llama.cpp_b200", "libb200qmm.so"))
    L.b200_flow_selftest_postponed_rope.restype = C.c_int
    assert L.b200_flow_selftest_postponed_rope() == 0

"""The Q8_K hand-over between phases of the persistent decode kernel (csrc/decode_flow.cu): a SwiGLU output is quantised to Q8_K
once per 256-block, by one designated CTA of the phase that produces it, and the mat-vec that reads it (ffn_down) loads those blocks
instead of polling the f32 vector and quantising it again in every CTA.

CPU: the host plan.  Every block has exactly one quantiser and that CTA owns the block's last row; plans that cannot give every block
one, consumers with a fused RMS_NORM and inputs that are not a SwiGLU output keep the f32 route; the slot pool still holds several
layers between two writes of a slot.
GPU: gate|up -> ffn_down as one launch is bit-identical to the same two phases launched as two programs, where the second one reads a
plain input and quantises it in its prologue; repeated launches are bit-identical."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "llama.cpp_b200", "libb200qmm.so")
Q4_K, Q6_K = 12, 14
POOL = 512 * 1024            # tagged slots of the ggml backend's pool (MEGA_LL_ELEMS) and of the C ABI's programs


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        pytest.skip("libb200qmm.so not built")
    L = C.CDLL(LIB)
    L.b200_flow_q8k_plan.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p]
    L.b200_flow_q8k_reuse.argtypes = [C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    return L


def q8k_plan(L, M, K_in, producer_mode=2, consumer_norm=False, grid=132):
    blk = (C.c_int * grid)()
    rc = L.b200_flow_q8k_plan(producer_mode, M, K_in, int(consumer_norm), grid, blk)
    return rc, list(blk)


def rows_of(M, grid, c):
    rq, rr = divmod(M, grid)
    rb = c * rq + min(c, rr)
    return rb, rb + rq + (1 if c < rr else 0)


# (SwiGLU rows M = ffn_down's K, gate|up input length): Llama-3-8B; its ffn_down K slices under -sm tensor x2 / x4 / x8 (the shapes
# test_flow_plan.py lists); Llama-3-70B under -sm tensor x8
SHAPES = [(14336, 4096), (14336 // 2, 4096), (14336 // 4, 4096), (14336 // 8, 4096), (3584, 8192)]


@pytest.mark.parametrize("M,K_in", SHAPES)
def test_every_block_has_one_quantiser_that_owns_its_last_row(lib, M, K_in):
    grid = 132
    rc, blk = q8k_plan(lib, M, K_in, grid=grid)
    assert rc == 1
    nb = M // 256
    owners = {}
    for c, b in enumerate(blk):
        if b < 0:
            continue
        assert b < nb and b not in owners, (c, b)
        owners[b] = c
    assert sorted(owners) == list(range(nb))
    spans = []
    for b, c in owners.items():
        rb, re = rows_of(M, grid, c)
        assert rb <= 256 * b + 255 < re                      # it polls rows of others only after writing its own
        spans.append(sum(1 for d in range(grid) if max(rows_of(M, grid, d)[0], 256 * b) < min(rows_of(M, grid, d)[1], 256 * b + 256)))
    if M == 14336:
        assert max(spans) == 4                                # a block's rows come from up to 4 CTAs at 108 - 109 rows per CTA


def test_plans_without_one_quantiser_per_block_keep_the_f32_route(lib):
    # 14336 rows on 56 CTAs: 256 per CTA, every CTA owns exactly one block; on 48 CTAs a CTA owns more than 256 rows and would have to
    # quantise two blocks
    rc, blk = q8k_plan(lib, 14336, 4096, grid=56)
    assert rc == 1 and sorted(blk) == list(range(56))
    rc, blk = q8k_plan(lib, 14336, 4096, grid=48)
    assert rc == 0 and all(b == -1 for b in blk)


def test_other_inputs_keep_the_f32_route(lib):
    assert q8k_plan(lib, 4096, 4096)[0] == 1
    rc, blk = q8k_plan(lib, 4096, 4096, consumer_norm=True)      # a fused RMS_NORM scales the whole vector before Q8_K rounding
    assert rc == 0 and all(b == -1 for b in blk)
    rc, blk = q8k_plan(lib, 4096, 4096, producer_mode=0)         # not a SwiGLU output
    assert rc == 0 and all(b == -1 for b in blk)
    assert q8k_plan(lib, 14336 + 128, 4096)[0] < 0               # ragged K: no mat-vec phase reads it at all


def test_slot_pool_holds_several_layers(lib):
    n_q8k, dist = C.c_int(0), C.c_int(0)
    assert lib.b200_flow_q8k_reuse(32, 14336, POOL, 132, C.byref(n_q8k), C.byref(dist)) == 0
    assert n_q8k.value == 32                                     # every ffn_down reads Q8_K blocks
    # a phase reads slots written at most 4 phases earlier (the residual of attn_output: the previous ffn_down's output); a slot is
    # rewritten only after many layers (5 phases each)
    assert dist.value >= 8 * 5, dist.value


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def host():
    import torch
    import llama_cpp_b200.host as h
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test without a GPU")
    assert h.device_count() >= 1, "libb200qmm.so sees no sm_90 device"
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("H,FF,M_down,t_down", [
    (4096, 14336, 4096, Q6_K), (4096, 14336, 4096, Q4_K),   # Llama-3-8B's two ffn_down types; a block spans up to 4 CTAs
    (4096, 1792, 4096, Q4_K),                               # K = 1792: 7 blocks
    (1024, 14336, 64, Q6_K),                                # 64 ffn_down rows: CTAs without rows in the consumer phase
])
def test_one_launch_matches_two(host, lib, H, FF, M_down, t_down):
    import torch
    from tools.gemv_sweep import blocks
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    assert q8k_plan(lib, FF, H, grid=grid)[0] == 1              # the one-launch program takes the Q8_K route on this device
    g = torch.Generator(device="cuda").manual_seed(FF + M_down + t_down)
    x = torch.randn(H, device="cuda", generator=g)
    nw = 1.0 + 0.1 * torch.randn(H, device="cuda", generator=g)
    gate, up, down = blocks(Q4_K, FF, H, g), blocks(Q4_K, FF, H, g), blocks(t_down, M_down, FF, g)
    resid = torch.randn(M_down, device="cuda", generator=g)

    def phases(act, y):
        return [dict(type=Q4_K, ws=[gate, up], x=x, norm_w=nw, eps=1e-5, mode=2, outs=[act]),
                dict(type=t_down, ws=[down], x=act, mode=1, residual=resid, outs=[y])]

    act2, y2 = torch.full((FF,), float("nan"), device="cuda"), torch.full((M_down,), float("nan"), device="cuda")
    p = phases(act2, y2)
    host.matvec_program(p[:1])
    host.matvec_program(p[1:])                                  # plain input: the prologue quantises the f32 vector
    torch.cuda.synchronize()
    ref_act, ref_y = act2.cpu().numpy(), y2.cpu().numpy()
    assert np.isfinite(ref_act).all() and np.isfinite(ref_y).all()
    for rep in range(3):
        act1, y1 = torch.full((FF,), float("nan"), device="cuda"), torch.full((M_down,), float("nan"), device="cuda")
        host.matvec_program(phases(act1, y1))
        torch.cuda.synchronize()
        a, y = act1.cpu().numpy(), y1.cpu().numpy()
        assert np.array_equal(a, ref_act), rep
        assert np.array_equal(y, ref_y), (rep, int((y != ref_y).sum()), float(np.abs(y - ref_y).max()))

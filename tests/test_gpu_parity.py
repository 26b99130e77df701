"""GPU parity tests (an H100, sm_90a): the CUDA path through the C ABI vs the oracle.

Bars
  dequant            bit-exact
  act quantisation   bit-exact (qs, d, bsums)
  mul_mat            |gpu - oracle| <= 4e-6 * sum_k |w_k x_k|  per output (fp32 reduction order only; the integer
                     parts are identical because the activations are the CPU's own Q8 integers)
  north-star bound   max-abs <= 1e-3 on O(1) outputs
"""
import os

import numpy as np
import pytest
import torch

from oracle.oracle import ALL_TYPES, BLOCK_ELEMS, Q4_0, Q4_K, Q6_K, Q8_0, Q8_K, TYPE_NAMES, act_type, random_blocks, row_bytes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def host():
    import llama_cpp_b200.host as h
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test without a GPU")
    assert h.device_count() >= 1, "libb200qmm.so sees no sm_90 device"
    return h


def tol(oracle, t, w, x):
    K = x.shape[-1]
    deq = np.stack([oracle.dequantize(t, w[m], K) for m in range(w.shape[0])])
    return np.abs(x)[:, None, :].__mul__(np.abs(deq)[None]).sum(-1)     # [N, M]


@pytest.mark.parametrize("t", ALL_TYPES)
def test_dequant_bit_exact(host, oracle, t):
    rng = np.random.default_rng(t)
    for K in (256, 4096):
        w = random_blocks(t, 33, K, rng)
        got = host.dequantize_rows(t, host.to_device_weights(w), K).cpu().numpy()
        want = np.stack([oracle.dequantize(t, w[m], K) for m in range(33)])
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), TYPE_NAMES[t]


@pytest.mark.parametrize("t", ALL_TYPES)
def test_dequant_golden(host, t):
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qmm_golden.npz"))
    n = TYPE_NAMES[t]
    got = host.dequantize_rows(t, host.to_device_weights(g[f"w_{n}"]), g[f"deq_{n}"].shape[1]).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), g[f"deq_{n}"].view(np.uint32))


@pytest.mark.parametrize("t", [Q4_0, Q4_K])
def test_act_quant_bit_exact(host, oracle, t):
    rng = np.random.default_rng(17)
    K = 4096
    x = rng.standard_normal((5, K)).astype(np.float32)
    x[1, :256] = 0.0                      # all-zero block
    x[2, 7] = -x[2, 300:556].max() * 9    # negative max-magnitude element
    x[3, :256] = np.where(np.arange(256) % 2 == 0, 1.0, -1.0)  # ties in |x| with both signs: first one wins
    x[4, :32] = np.arange(32) + 0.5       # exact .5 ties
    qs, d, bs, _ = host.quantize_act(t, torch.from_numpy(x).cuda())
    qs, d, bs = qs.cpu().numpy(), d.cpu().numpy(), bs.cpu().numpy()
    for i in range(x.shape[0]):
        a = oracle.quantize_act(t, x[i])
        if act_type(t) == Q8_K:
            b = a.reshape(K // 256, 292)
            assert np.array_equal(qs[i], b[:, 4:260].copy().view(np.int8).reshape(-1)), i
            assert np.array_equal(d[i].view(np.uint32), b[:, :4].copy().view(np.uint32).reshape(-1)), i
            assert np.array_equal(bs[i], b[:, 260:].copy().view(np.int16).reshape(-1)), i
        else:
            b = a.reshape(K // 32, 34)
            assert np.array_equal(qs[i], b[:, 2:].copy().view(np.int8).reshape(-1)), i
            assert np.array_equal(d[i], b[:, :2].copy().view(np.float16).astype(np.float32).reshape(-1)), i
            assert np.array_equal(bs[i], qs[i].reshape(-1, 32).astype(np.int32).sum(1).astype(np.int16)), i


def test_act_quant_golden(host):
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qmm_golden.npz"))
    x = g["x"]
    qs, d, bs, _ = host.quantize_act(Q4_K, torch.from_numpy(x).cuda())
    want = g["act_q4_K"].reshape(x.shape[0], -1, 292)
    assert np.array_equal(qs.cpu().numpy(), want[:, :, 4:260].copy().view(np.int8).reshape(x.shape[0], -1))
    assert np.array_equal(d.cpu().numpy().view(np.uint32), want[:, :, :4].copy().view(np.uint32).reshape(x.shape[0], -1))


@pytest.mark.parametrize("t", ALL_TYPES)
@pytest.mark.parametrize("N", [1, 2, 3, 5, 8])
def test_mul_mat_decode_regime(host, oracle, t, N):
    rng = np.random.default_rng(1000 * t + N)
    for (M, K) in ((16, 256), (37, 2304), (130, 4352)):
        w = random_blocks(t, M, K, rng)
        x = rng.standard_normal((N, K)).astype(np.float32)
        got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
        want = oracle.mul_mat(t, w, x)
        bound = 4e-6 * tol(oracle, t, w, x) + 1e-30
        err = np.abs(got - want)
        assert (err <= bound).all(), (TYPE_NAMES[t], N, M, K, float(err.max()), float((err / bound).max()))
        assert err.max() <= 1e-3


@pytest.mark.parametrize("t", ALL_TYPES)
def test_mul_mat_llama_shapes_vs_reference(host, oracle, ref, t):
    """Llama-3-8B shapes, weights quantised by the reference's own quantiser, checked against the REFERENCE's
    compiled CPU kernels (oracle/_ref) -- the north-star tolerance: max-abs <= 1e-3."""
    rng = np.random.default_rng(5 + t)
    M, K = 512, 4096
    w = ref.quantize_weights(t, (rng.standard_normal((M, K)) * 0.02).astype(np.float32))
    x = rng.standard_normal((1, K)).astype(np.float32)
    got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
    want_ref = ref.mul_mat(t, w, x, simd=(t not in (Q4_0, Q8_0)))   # Q8_0 activations: compare with the _ref rounding
    want_orc = oracle.mul_mat(t, w, x)
    assert np.abs(got - want_ref).max() <= 1e-3
    assert np.abs(got - want_orc).max() <= 1e-4
    assert np.abs(want_ref).max() > 0.5


@pytest.mark.parametrize("t", ALL_TYPES)
def test_first_generation_kernel_still_matches(host, oracle, t):
    """gemv.cu (variant 1) stays in the library as the general fallback; keep it parity-green."""
    rng = np.random.default_rng(4242 + t)
    host.lib().b200_set_gemv_variant(1)
    try:
        for (M, K, N) in ((37, 2304, 1), (130, 4352, 3)):
            w = random_blocks(t, M, K, rng)
            x = rng.standard_normal((N, K)).astype(np.float32)
            got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
            want = oracle.mul_mat(t, w, x)
            assert (np.abs(got - want) <= 4e-6 * tol(oracle, t, w, x) + 1e-30).all()
    finally:
        host.lib().b200_set_gemv_variant(2)


@pytest.mark.parametrize("t", [Q4_K, Q6_K])
def test_partial_row_groups_and_k_steps(host, oracle, t):
    """gemv2 works on groups of 4 rows x 8 blocks: M % 4 != 0 and (K/256) % 8 != 0 must be masked correctly."""
    rng = np.random.default_rng(99 + t)
    for (M, K) in ((1, 256), (2, 768), (3, 2816), (5, 11008 // 256 * 256), (1030, 512)):
        w = random_blocks(t, M, K, rng)
        x = rng.standard_normal((1, K)).astype(np.float32)
        got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
        want = oracle.mul_mat(t, w, x)
        assert (np.abs(got - want) <= 4e-6 * tol(oracle, t, w, x) + 1e-30).all(), (t, M, K)


@pytest.mark.parametrize("t", [Q4_K, 13, Q6_K])
def test_fused_matvec_modes(host, oracle, t):
    """gemv3 through the C ABI: fused RMS_NORM+quantise prologue, 3-matrix launch, residual and SwiGLU epilogues, against
    the oracle fed with the same normalised vector (computed here in float64->float32 exactly as ggml's RMS_NORM + MUL)."""
    rng = np.random.default_rng(300 + t)
    K = 1024
    x = rng.standard_normal(K).astype(np.float32)
    nw = (1.0 + 0.1 * rng.standard_normal(K)).astype(np.float32)
    eps = np.float32(1e-5)
    mean = np.float32(np.sum((x * x).astype(np.float64)) / K)
    scale = np.float32(1.0) / np.sqrt(mean + eps, dtype=np.float32)
    xn = ((x * scale).astype(np.float32) * nw).astype(np.float32)
    xd, nwd = torch.from_numpy(x).cuda(), torch.from_numpy(nw).cuda()
    ws = [random_blocks(t, M, K, rng) for M in (96, 40, 40)]
    wd = [host.to_device_weights(w) for w in ws]
    # mode 0, three matrices, with norm
    outs = host.fused_matvec(t, wd, xd, norm_w=nwd, eps=float(eps), mode=0)
    for w, o in zip(ws, outs):
        want = oracle.mul_mat(t, w, xn[None])[0]
        assert (np.abs(o.cpu().numpy() - want) <= 4e-6 * tol(oracle, t, w, xn[None])[0] + 1e-30).all()
    # mode 1, residual, no norm
    res = rng.standard_normal(96).astype(np.float32)
    out = host.fused_matvec(t, wd[:1], xd, mode=1, residual=[torch.from_numpy(res).cuda()])[0].cpu().numpy()
    want = oracle.mul_mat(t, ws[0], x[None])[0] + res
    assert (np.abs(out - want) <= 4e-6 * tol(oracle, t, ws[0], x[None])[0] + 1e-6).all()
    # mode 2, SwiGLU pair with norm
    out = host.fused_matvec(t, wd[1:3], xd, norm_w=nwd, eps=float(eps), mode=2)[0].cpu().numpy()
    g = oracle.mul_mat(t, ws[1], xn[None])[0]
    u = oracle.mul_mat(t, ws[2], xn[None])[0]
    want = (g / (1.0 + np.exp(-g))) * u
    assert np.abs(out - want).max() <= 1e-5 * max(1.0, float(np.abs(want).max()))


def test_matvec_program_matches_separate_launches(host):
    """The persistent dataflow decode kernel on a two-"layer" chain of fused mat-vecs with Llama-like dependencies (norm + q|k|v
    with a Q6_K v, o + residual, norm + gate|up SwiGLU, down (Q6_K) + residual): every phase reads what the previous phase
    wrote, across CTAs, through tagged slots -- no barrier.  Each phase is checked against ONE b200_fused_matvec launch fed with the
    program's own inputs of that phase (the plain copies every phase also writes): same integers, only the fp32 order of the
    row reduction differs.  Repeated launches must be bit-identical (the kernel is deterministic whatever the timing)."""
    g = torch.Generator(device="cuda").manual_seed(17)
    from tools.gemv_sweep import blocks
    H, FF = 1024, 7936                     # FF: 31 blocks per row (one k-segment, a ragged warp step)
    eps = 1e-5

    def mk(t, M, K):
        return blocks(t, M, K, g)

    layers = []
    for _ in range(2):
        layers.append(dict(nw1=1.0 + 0.1 * torch.randn(H, device="cuda", generator=g), nw2=1.0 + 0.1 * torch.randn(H, device="cuda", generator=g),
                           q=mk(Q4_K, H, H), k=mk(Q4_K, 256, H), v=mk(Q6_K, 256, H), o=mk(Q4_K, H, H),
                           gate=mk(Q4_K, FF, H), up=mk(Q4_K, FF, H), down=mk(Q6_K, H, FF)))
    x0 = torch.randn(H, device="cuda", generator=g)

    def build():
        phases, bufs = [], []
        cur = x0.clone()
        for L in layers:
            q, k, v = (torch.zeros(n, device="cuda") for n in (H, 256, 256))
            attn_in = q                                     # stands in for attention: o-proj consumes q directly
            ffn_inp = torch.zeros(H, device="cuda")
            act = torch.zeros(FF, device="cuda")
            nxt = torch.zeros(H, device="cuda")
            phases += [dict(types=[Q4_K, Q4_K, Q6_K], ws=[L["q"], L["k"], L["v"]], x=cur, norm_w=L["nw1"], eps=eps, mode=0, outs=[q, k, v]),
                       dict(type=Q4_K, ws=[L["o"]], x=attn_in, mode=1, residual=cur, outs=[ffn_inp]),
                       dict(type=Q4_K, ws=[L["gate"], L["up"]], x=ffn_inp, norm_w=L["nw2"], eps=eps, mode=2, outs=[act]),
                       dict(type=Q6_K, ws=[L["down"]], x=act, mode=1, residual=ffn_inp, outs=[nxt])]
            bufs += [q, k, v, ffn_inp, act, nxt]
            cur = nxt
        return phases, bufs

    runs = []
    for rep in range(4):                                    # repeated launches: the epoch moves on, nothing is reset
        phases, bufs = build()
        host.matvec_program(phases)
        torch.cuda.synchronize()
        runs.append([b.cpu().numpy() for b in bufs])
        for a in runs[-1]:
            assert np.isfinite(a).all()
        for i, (a, b) in enumerate(zip(runs[-1], runs[0])):
            assert np.array_equal(a, b), (rep, i, float(np.abs(a - b).max()))
    # phase by phase against the stand-alone kernel, teacher-forced with the program's own intermediate vectors
    worst = 0.0
    for p in phases:
        ts = p["types"] if "types" in p else [p["type"]] * len(p["ws"])
        groups = [[0, 1], [2]] if len(set(ts)) > 1 else [list(range(len(ts)))]     # the stand-alone kernel takes one type per launch
        if p["mode"] == 2:
            groups = [[0, 1]]
        for grp in groups:
            outs_ref = [torch.empty_like(p["outs"][0 if p["mode"] == 2 else j]) for j in (grp[:1] if p["mode"] == 2 else grp)]
            host.fused_matvec(ts[grp[0]], [p["ws"][j] for j in grp], p["x"], norm_w=p.get("norm_w"), eps=eps, mode=p["mode"],
                              residual=[p["residual"]] if p.get("residual") is not None else None, outs=outs_ref)
            torch.cuda.synchronize()
            for j, o in zip(grp, outs_ref):
                got = p["outs"][0 if p["mode"] == 2 else j]
                err = (got - o).abs().max().item()
                worst = max(worst, err / max(1.0, o.abs().max().item()))
                assert err <= 2e-5 * max(1.0, o.abs().max().item()), (p["mode"], j, err)
    print(f"program vs stand-alone launches: worst relative difference {worst:.2e}")
    # a long activation (ffn_down of Llama-3-8B: K = 14336, a row is split over two warps), fewer rows than CTAs
    K2 = 14336
    for t in (Q4_K, Q6_K):
        for M2 in (72, 600):
            w = mk(t, M2, K2)
            x = torch.randn(K2, device="cuda", generator=g)
            out = torch.empty(M2, device="cuda")
            host.matvec_program([dict(type=t, ws=[w], x=x, mode=0, outs=[out])])
            ref = host.mul_mat(t, w, x[None])[0]
            torch.cuda.synchronize()
            err = (out - ref).abs().max().item()
            assert err <= 2e-5 * max(1.0, ref.abs().max().item()), (t, M2, err)
    # a long single-matrix phase (an output head): hundreds of ring pieces per CTA, every slot reused many times while the weight stream
    # is the bottleneck -- the consumer warps run ahead of the copies
    for t in (Q4_K, Q6_K):
        w = mk(t, 33000, 4096)
        x = torch.randn(4096, device="cuda", generator=g)
        out = torch.empty(33000, device="cuda")
        host.matvec_program([dict(type=t, ws=[w], x=x, mode=0, outs=[out])])
        ref = host.mul_mat(t, w, x[None])[0]
        torch.cuda.synchronize()
        err = (out - ref).abs().max().item()
        assert err <= 2e-5 * max(1.0, ref.abs().max().item()), (t, 33000, err)


def test_mul_mat_rows_not_16B_multiples(host, oracle):
    # Q4_0 with K = 2880 (test-backend-ops.cpp:9167): row bytes 1620, rows only 4-byte aligned
    rng = np.random.default_rng(9)
    M, K = 67, 2880
    w = random_blocks(Q4_0, M, K, rng)
    x = rng.standard_normal((2, K)).astype(np.float32)
    got = host.mul_mat(Q4_0, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
    want = oracle.mul_mat(Q4_0, w, x)
    assert (np.abs(got - want) <= 4e-6 * tol(oracle, Q4_0, w, x) + 1e-30).all()


def test_mul_mat_strided_rows_and_empty(host, oracle):
    rng = np.random.default_rng(21)
    M, K = 40, 512
    rb = row_bytes(Q6_K, K)
    wide = np.zeros((M, 2 * rb), np.uint8)
    w = random_blocks(Q6_K, M, K, rng)
    wide[:, :rb] = w
    wd = host.to_device_weights(wide)[:, :rb]           # row stride = 2*rb
    x = rng.standard_normal((1, K)).astype(np.float32)
    got = host.mul_mat(Q6_K, wd, torch.from_numpy(x).cuda()).cpu().numpy()
    assert (np.abs(got - oracle.mul_mat(Q6_K, w, x)) <= 4e-6 * tol(oracle, Q6_K, w, x) + 1e-30).all()
    # empty inputs are no-ops
    out = host.mul_mat(Q6_K, wd[:0], torch.from_numpy(x).cuda())
    assert out.shape == (1, 0)


@pytest.mark.parametrize("N", [9, 17, 64])
def test_mul_mat_more_than_8_columns(host, oracle, N):
    rng = np.random.default_rng(N)
    M, K = 96, 1024
    w = random_blocks(Q4_K, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    got = host.mul_mat(Q4_K, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
    want = oracle.mul_mat(Q4_K, w, x)
    assert np.abs(got - want).max() <= 1e-3
    assert (np.abs(got - want) <= 2e-5 * tol(oracle, Q4_K, w, x) + 1e-30).all()


GEMM_SHAPES = [(128, 256, 16), (130, 512, 9), (256, 1024, 128), (300, 2304, 200), (128, 4096, 130), (256, 512, 400)]


@pytest.mark.parametrize("M,K,N", GEMM_SHAPES)
@pytest.mark.parametrize("t", [Q4_K, 13, Q6_K])
def test_gemm_tcgen05_matches_oracle(host, oracle, t, M, K, N):
    """Prefill regime (wgmma on integer operands + per-block fp32 rescale) vs the oracle: the bound is 1.5x the decode
    GEMV's -- the fp32 combine order differs from the CPU's, and a block's integer sum above 2^24 is accumulated in fp32.
    Shapes cover ragged M and N tiles, one and many K blocks, a zero activation block.  Two inputs per shape: random
    blocks, and saturated blocks (oracle.saturated_blocks: every weight field at its extreme, every Q8_K integer +-127,
    block sums up to 1.3e8)."""
    from oracle.oracle import constant_sign_blocks, saturated_blocks
    rng = np.random.default_rng(900 + t + M + K + N)
    host.lib().b200_set_mul_mat_path(2)
    try:
        for kind in ("random", "saturated"):
            if kind == "random":
                w = random_blocks(t, M, K, rng)
                x = rng.standard_normal((N, K)).astype(np.float32)
                x[0, :256] = 0.0
            else:
                w = saturated_blocks(t, M, K, rng)
                x = constant_sign_blocks(N, K, rng)
            got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
            want = oracle.mul_mat(t, w, x)
            bound = 6e-6 * tol(oracle, t, w, x) + 1e-30
            err = np.abs(got - want)
            assert np.isfinite(got).all()
            ratio = float((err / bound).max())
            print(f"gemm {TYPE_NAMES[t]} {M}x{K}x{N} {kind}: worst err/bound {ratio:.3f}")
            assert (err <= bound).all(), (t, M, K, N, kind, float(err.max()), ratio, float(np.abs(want).max()))
    finally:
        host.lib().b200_set_mul_mat_path(0)


@pytest.mark.parametrize("t", [Q4_0, Q8_0])
def test_gemm_legacy_tcgen05_matches_oracle(host, oracle, t):
    """Q4_0 / Q8_0 prefill GEMM on wgmma (gemm_legacy_wgmma.cu): the per-32 scales are folded into hi/lo fp16 operand pairs and
    three MMAs per k-slice accumulate in fp32 over the whole K.  Against the oracle (the CPU's Q8_0 activation integers, exact integer
    block sums, fp32 combine) only fp32 rounding / order differs: same bound as the K-quant GEMM.  Shapes cover ragged M and N tiles,
    one and many 256-weight supersteps, a zero activation block."""
    rng = np.random.default_rng(1900 + t)
    host.lib().b200_set_mul_mat_path(2)
    try:
        for (M, K, N) in GEMM_SHAPES:
            w = random_blocks(t, M, K, rng)
            x = rng.standard_normal((N, K)).astype(np.float32)
            x[0, :256] = 0.0
            got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
            want = oracle.mul_mat(t, w, x)
            bound = 6e-6 * tol(oracle, t, w, x) + 1e-30
            err = np.abs(got - want)
            assert np.isfinite(got).all()
            assert (err <= bound).all(), (t, M, K, N, float(err.max()), float((err / bound).max()), float(np.abs(want).max()))
    finally:
        host.lib().b200_set_mul_mat_path(0)


@pytest.mark.parametrize("t", [Q4_0, Q8_0])
def test_gemm_legacy_reference_quantised_weights(host, ref, t):
    """Llama-shaped legacy-format GEMM with weights from the reference quantiser, vs the reference's own CPU kernels: <= 1e-3 max-abs."""
    rng = np.random.default_rng(78)
    M, K, N = 512, 4096, 96
    w = ref.quantize_weights(t, (rng.standard_normal((M, K)) * 0.02).astype(np.float32))
    x = rng.standard_normal((N, K)).astype(np.float32)
    got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
    want = ref.mul_mat(t, w, x, simd=True)
    assert np.abs(got - want).max() <= 1e-3, float(np.abs(got - want).max())
    assert np.abs(want).max() > 0.5


def test_gemm_tcgen05_reference_quantised_weights(host, oracle, ref):
    """Llama-shaped GEMM with weights from the reference quantiser, vs the reference's own CPU kernels: <= 1e-3 max-abs."""
    rng = np.random.default_rng(77)
    M, K, N = 512, 4096, 96
    w = ref.quantize_weights(Q4_K, (rng.standard_normal((M, K)) * 0.02).astype(np.float32))
    x = rng.standard_normal((N, K)).astype(np.float32)
    got = host.mul_mat(Q4_K, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()
    want = ref.mul_mat(Q4_K, w, x, simd=True)
    assert np.abs(got - want).max() <= 1e-3, float(np.abs(got - want).max())
    assert np.abs(want).max() > 0.5


@pytest.mark.parametrize("t", [Q4_K, Q8_0])
@pytest.mark.parametrize("nb1_is_one", [True, False])
def test_mul_mat_id(host, oracle, t, nb1_is_one):
    """b200_mul_mat_id (the routed GEMV) per element at the GEMV bar, 4e-6 sum_k |w_k x_k|."""
    rng = np.random.default_rng(31)
    E, M, K, T, n_used = 8, 48, 512, 5, 2
    w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
    nb1 = 1 if nb1_is_one else n_used
    b = rng.standard_normal((T, nb1, K)).astype(np.float32)
    ids = rng.integers(0, E, size=(T, n_used)).astype(np.int32)
    wd = host.to_device_weights(w.reshape(E * M, -1)).view(E, M, -1)
    got = host.mul_mat_id(t, wd, torch.from_numpy(b).cuda(), torch.from_numpy(ids).cuda()).cpu().numpy()
    want = oracle.mul_mat_id(t, w, b, ids)
    assert np.abs(got - want).max() <= 1e-4
    for tkn in range(T):
        for s in range(n_used):
            col = b[tkn, s % nb1][None]
            bound = 4e-6 * tol(oracle, t, w[ids[tkn, s]], col)[0] + 1e-30
            assert (np.abs(got[tkn, s] - want[tkn, s]) <= bound).all(), (tkn, s, float((np.abs(got[tkn, s] - want[tkn, s]) / bound).max()))


@pytest.mark.parametrize("t,M,K,N", [(Q4_K, 14336, 4096, 2048), (Q6_K, 4096, 14336, 2048), (Q4_0, 11008, 4096, 2048), (Q6_K, 128256, 4096, 1)])
def test_bench_shapes_sampled_rows_and_columns(host, oracle, t, M, K, N):
    """Parity AT the benchmarked shapes (the prefill GEMMs of pp2048: ffn_gate Q4_K, ffn_down Q6_K; Llama-2-7B's Q4_0 ffn_up; the 128256-row
    Q6_K output head of a decode step): the full-size product is computed on the device and 48 sampled weight rows x 12 sampled token columns
    are checked against the oracle (activation quantisation is per column and a row's dot product is independent of the other rows, so
    the oracle on the sub-problem is the oracle's answer for those elements of the full problem).  Bound: as for the small shapes."""
    rng = np.random.default_rng(4000 + t + M % 97)
    w = random_blocks(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    got = host.mul_mat(t, host.to_device_weights(w), torch.from_numpy(x).cuda()).cpu().numpy()          # [N, M]
    assert got.shape == (N, M) and np.isfinite(got).all()
    rows = np.unique(np.concatenate([[0, 1, 127, 128, M - 1], rng.integers(0, M, size=43)]))
    cols = np.unique(np.concatenate([[0, N - 1], rng.integers(0, N, size=10)])) if N > 1 else np.array([0])
    ws, xs = np.ascontiguousarray(w[rows]), np.ascontiguousarray(x[cols])
    want = oracle.mul_mat(t, ws, xs)                                                                     # [len(cols), len(rows)]
    sub = got[np.ix_(cols, rows)]
    err = np.abs(sub - want)
    bound = 6e-6 * tol(oracle, t, ws, xs) + 1e-30
    assert (err <= bound).all(), (TYPE_NAMES[t], M, K, N, float(err.max()), float((err / bound).max()))
    assert err.max() <= 1e-3


def test_linearity_and_permutation_properties_full_size(host):
    """Size-independent properties at a full Llama-3-8B shape (oracle too slow there): scaling the activations by 2
    scales the Q8_K scale exactly (power of two) so the output doubles bit-exactly; permuting weight rows permutes
    outputs."""
    M, K = 14336, 4096
    g = torch.Generator(device="cuda").manual_seed(3)
    w = torch.randint(0, 256, (M, row_bytes(Q4_K, K)), dtype=torch.uint8, device="cuda", generator=g)
    wv = w.view(M, K // 256, 144)
    wv[:, :, 1] = 0x1C
    wv[:, :, 3] = 0x1C                     # d, dmin ~ 2^-8: finite
    x = torch.randn((1, K), device="cuda", generator=g)
    y1 = host.mul_mat(Q4_K, w, x)
    y2 = host.mul_mat(Q4_K, w, 2 * x)
    assert torch.equal(2 * y1, y2)
    perm = torch.randperm(M, device="cuda", generator=g)
    y3 = host.mul_mat(Q4_K, w[perm].contiguous(), x)
    assert torch.equal(y3, y1[:, perm])
    assert torch.isfinite(y1).all()


def test_host_buffer_entry_point(host, oracle):
    rng = np.random.default_rng(77)
    M, K = 64, 1024
    w = random_blocks(Q4_K, M, K, rng)
    hm = host.HostMulMat(Q4_K, host.to_device_weights(w), 1, K)
    x = rng.standard_normal((1, K)).astype(np.float32)
    hm.x_host.copy_(torch.from_numpy(x))
    got = hm().numpy().copy()
    assert np.abs(got - oracle.mul_mat(Q4_K, w, x)).max() <= 1e-4

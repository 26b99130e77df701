"""CPU-only: pin the oracle (oracle/qmm_oracle.c) against
  (1) the committed golden vectors generated from the reference's own compiled code, and
  (2) the reference itself (oracle/_ref) on fresh seeded inputs, when it is present.
Bars: dequant / activation quantisation / integer dot pieces bit-exact; fp32 dot within 2e-6 relative of the
sum of |terms| (only the fp32 reduction order / FMA contraction differs)."""
import os

import numpy as np
import pytest

from oracle.oracle import ALL_TYPES, BLOCK_BYTES, BLOCK_ELEMS, Q4_K, Q5_K, Q6_K, Q8_K, TYPE_NAMES, act_type, random_blocks, row_bytes

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qmm_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_fp16_roundtrip_all_halves(oracle):
    # every finite half converts exactly to fp32 and back
    hs = np.arange(0, 1 << 16, dtype=np.uint32)
    hs = hs[(hs & 0x7C00) != 0x7C00]
    want = hs.astype(np.uint16).view(np.float16).astype(np.float32)
    got = np.array([oracle.lib.orc_fp16_to_fp32(int(h)) for h in hs[::7]], dtype=np.float32)
    assert np.array_equal(got.view(np.uint32), want[::7].view(np.uint32))
    back = np.array([oracle.lib.orc_fp32_to_fp16(float(v)) for v in want[::7]], dtype=np.uint16)
    assert np.array_equal(back, hs[::7].astype(np.uint16))


def test_fp32_to_fp16_rounding_matches_numpy(oracle):
    rng = np.random.default_rng(7)
    v = np.concatenate([rng.standard_normal(4000) * 10.0 ** rng.integers(-9, 5, 4000), [0.0, 65504.0, 65519.9, 65520.0, 2.0 ** -25, 2.0 ** -24, 5.96e-8]]).astype(np.float32)
    got = np.array([oracle.lib.orc_fp32_to_fp16(float(x)) for x in v], dtype=np.uint16)
    with np.errstate(over="ignore"):
        want = v.astype(np.float16).view(np.uint16)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("t", ALL_TYPES)
def test_dequant_matches_golden_bit_exact(oracle, golden, t):
    n = TYPE_NAMES[t]
    w, deq = golden[f"w_{n}"], golden[f"deq_{n}"]
    for m in range(w.shape[0]):
        got = oracle.dequantize(t, w[m], deq.shape[1])
        assert np.array_equal(got.view(np.uint32), deq[m].view(np.uint32)), (n, m)


@pytest.mark.parametrize("t", ALL_TYPES)
def test_act_quant_matches_golden_bit_exact(oracle, golden, t):
    n = TYPE_NAMES[t]
    x, acts = golden["x"], golden[f"act_{n}"]
    for i in range(x.shape[0]):
        got = oracle.quantize_act(t, x[i])
        want = acts[i].copy()
        if act_type(t) == Q8_K:
            # reference leaves bsums of an all-zero block unwritten (ggml-quants.c:2782-2787); compare d and qs only there
            for b in range(x.shape[1] // 256):
                if not x[i, 256 * b:256 * (b + 1)].any():
                    want[292 * b + 260:292 * (b + 1)] = 0
        assert np.array_equal(got, want), (n, i)


@pytest.mark.parametrize("t", ALL_TYPES)
def test_vec_dot_matches_golden(oracle, golden, t):
    n = TYPE_NAMES[t]
    w, acts, dots, deq, x = golden[f"w_{n}"], golden[f"act_{n}"], golden[f"dot_{n}"], golden[f"deq_{n}"], golden["x"]
    K = deq.shape[1]
    for i in range(acts.shape[0]):
        for m in range(w.shape[0]):
            got = oracle.vec_dot(t, K, w[m], acts[i])
            scale = float(np.abs(deq[m] * x[i]).sum()) + 1e-30
            assert abs(got - dots[i, m]) <= 2e-6 * scale, (n, i, m, got, dots[i, m])


@pytest.mark.parametrize("t", ALL_TYPES)
def test_against_reference_fresh_inputs(oracle, ref, t):
    """Random valid blocks (all code/scale bit patterns), ragged K, vs the reference compiled here."""
    rng = np.random.default_rng(100 + t)
    for K in (256, 512, 2304):
        if K % BLOCK_ELEMS[t]:
            continue
        w = random_blocks(t, 5, K, rng)
        x = rng.uniform(-2, 2, size=(2, K)).astype(np.float32)
        for m in range(w.shape[0]):
            a = oracle.dequantize(t, w[m], K)
            b = ref.dequantize(t, w[m], K)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        for i in range(2):
            qa, qb = oracle.quantize_act(t, x[i]), ref.quantize_act(t, x[i])
            assert np.array_equal(qa, qb)
            for m in range(w.shape[0]):
                got, want = oracle.vec_dot(t, K, w[m], qa), ref.vec_dot(t, K, w[m], qb)
                scale = float(np.abs(ref.dequantize(t, w[m], K) * x[i]).sum()) + 1e-30
                assert abs(got - want) <= 2e-6 * scale


@pytest.mark.parametrize("t", ALL_TYPES)
def test_simd_and_generic_reference_agree_with_oracle(oracle, ref, t):
    """The AVX2 kernels the reference actually runs differ from its generic code only in fp32 order."""
    rng = np.random.default_rng(5)
    K = 1024
    w = ref.quantize_weights(t, (rng.standard_normal((4, K)) * 0.02).astype(np.float32))
    x = rng.standard_normal((1, K)).astype(np.float32)
    a = oracle.quantize_act(t, x[0])
    for m in range(4):
        s = ref.vec_dot(t, K, w[m], a, generic=False)
        g = oracle.vec_dot(t, K, w[m], a)
        assert abs(s - g) <= 5e-6 * float(np.abs(oracle.dequantize(t, w[m], K) * x[0]).sum())


@pytest.mark.parametrize("t", ALL_TYPES)
def test_mul_mat_is_quantize_then_dot(oracle, t):
    rng = np.random.default_rng(11)
    M, N, K = 7, 3, 512
    w = random_blocks(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    out = oracle.mul_mat(t, w, x)
    assert out.shape == (N, M)
    for n in range(N):
        a = oracle.quantize_act(t, x[n])
        for m in range(M):
            assert out[n, m] == np.float32(oracle.vec_dot(t, K, w[m], a))
    # close to the unquantised-activation product (sanity of the whole chain): Q8 noise ~1e-2 relative
    deq = np.stack([oracle.dequantize(t, w[m], K) for m in range(M)])
    exact = x @ deq.T
    assert np.abs(out - exact).max() <= 2e-2 * np.abs(exact).max() + 1e-3


def test_mul_mat_id_routes_rows(oracle):
    from oracle.oracle import Q4_K
    rng = np.random.default_rng(3)
    E, M, K, T, n_used = 4, 6, 256, 5, 2
    w = np.stack([random_blocks(Q4_K, M, K, rng) for _ in range(E)])
    b = rng.standard_normal((T, 1, K)).astype(np.float32)   # broadcast activations (nb1 = 1)
    ids = rng.integers(0, E, size=(T, n_used)).astype(np.int32)
    out = oracle.mul_mat_id(Q4_K, w, b, ids)
    for tkn in range(T):
        for s in range(n_used):
            want = oracle.mul_mat(Q4_K, w[ids[tkn, s]], b[tkn])
            assert np.array_equal(out[tkn, s], want[0])


@pytest.mark.parametrize("nb1_is_one", [True, False])
@pytest.mark.parametrize("t", ALL_TYPES)
def test_mul_mat_id_matches_ggml_cpu_mul_mat_id(oracle, ref, t, nb1_is_one):
    """oracle.mul_mat_id against ggml_mul_mat_id on the reference's CPU backend, with the ids as llama builds them (the first n_used
    rows of an [n_expert, T] tensor) and one token routed to the same expert twice.  Weights from the reference quantiser, O(1) outputs:
    max-abs <= 1e-3, the bar of the reference-shaped mat-mul tests (the CPU backend quantises Q8_0 activations with its SIMD rounding,
    the oracle with the _ref rounding; they differ at ties only).  K-quants share the Q8_K integers and differ in fp32 order only:
    also <= 5e-6 sum_k |w_k x_k| per element."""
    rng = np.random.default_rng(40 + t + 7 * nb1_is_one)
    E, M, K, T, n_used = 4, 24, 4096, 6, 2
    w = np.stack([ref.quantize_weights(t, (rng.standard_normal((M, K)) * 0.02).astype(np.float32)) for _ in range(E)])
    nb1 = 1 if nb1_is_one else n_used
    b = rng.standard_normal((T, nb1, K)).astype(np.float32)
    ids = np.stack([rng.permutation(E)[:n_used] for _ in range(T)]).astype(np.int32)
    ids[2] = [3, 3]                                           # the same expert in both slots of one token
    want = ref.mul_mat_id(t, w, b, ids)
    got = oracle.mul_mat_id(t, w, b, ids)
    assert np.isfinite(want).all() and np.abs(want).max() > 0.5
    assert np.abs(got - want).max() <= 1e-3, float(np.abs(got - want).max())
    if t in (Q4_K, Q5_K, Q6_K):
        deq = np.stack([np.stack([oracle.dequantize(t, w[e, m], K) for m in range(M)]) for e in range(E)])        # [E, M, K]
        cols = b[np.arange(T)[:, None], np.arange(n_used)[None] % nb1]                                             # [T, n_used, K]
        scale = np.einsum("tsk,tsmk->tsm", np.abs(cols), np.abs(deq[ids]))
        assert (np.abs(got - want) <= 5e-6 * scale).all()
    assert np.array_equal(got[2, 0], got[2, 1]) == (nb1 == 1)


def test_empty_and_sizes(oracle):
    for t in ALL_TYPES:
        assert row_bytes(t, 0) == 0
        assert oracle.lib.orc_dequantize_row(t, None, None, 0) == 0
        assert oracle.lib.orc_dequantize_row(t, None, None, BLOCK_ELEMS[t] + 1) == -1  # ragged K is rejected, as ggml asserts
        assert oracle.lib.orc_row_bytes(t, 4096) == 4096 // BLOCK_ELEMS[t] * BLOCK_BYTES[t]


# ---- attention and ROPE: the float64 restatements the GPU attention tests compare against, pinned to ggml's own CPU code

def _fa_case(rng, B, H, Hkv, N, n_kv, D, mask_kind):
    q = rng.standard_normal((B, H, N, D)).astype(np.float32)
    k = rng.standard_normal((B, Hkv, n_kv, D)).astype(np.float16)
    v = rng.standard_normal((B, Hkv, n_kv, D)).astype(np.float16)
    if mask_kind is None:
        return q, k, v, None
    m2 = H if mask_kind == "per_head" else 1
    m = np.where(rng.random((B, m2, N, n_kv)) < 0.3, -np.inf, rng.uniform(-2, 2, (B, m2, N, n_kv))).astype(np.float16)
    m[:, :, 1, :] = -np.inf                                   # a row with every key masked: 0, not NaN
    return q, k, v, m


@pytest.mark.parametrize("B,H,Hkv,N,n_kv,D,mask_kind,softcap", [
    (1, 4, 4, 3, 17, 64, None, 0.0),
    (2, 8, 2, 5, 37, 64, "broadcast", 0.0),                   # GQA 4, one mask plane for every head
    (1, 8, 1, 4, 70, 128, "per_head", 0.0),                   # GQA 8, mask ne2 = H
    (2, 4, 2, 6, 129, 128, "broadcast", 30.0),                # softcap
    (1, 2, 1, 2, 300, 256, "per_head", 0.0),
])
def test_attention_f64_matches_ggml_cpu_flash_attn(ref, B, H, Hkv, N, n_kv, D, mask_kind, softcap):
    """The restatement against ggml_flash_attn_ext on the reference's CPU backend, which accumulates V in f16: <= 2e-3 max|v|."""
    from oracle.oracle import attention_f64
    rng = np.random.default_rng(N * 1000 + n_kv)
    q, k, v, m = _fa_case(rng, B, H, Hkv, N, n_kv, D, mask_kind)
    scale = 1.0 / np.sqrt(D)
    want = ref.flash_attn_ext(q, k, v, m, scale, softcap)
    got = attention_f64(q, k, v, m, scale, softcap)
    assert np.isfinite(want).all() and np.isfinite(got).all()
    assert np.abs(got - want).max() <= 2e-3 * np.abs(v.astype(np.float32)).max()
    if m is not None:
        assert (got[:, 1] == 0).all() and (want[:, 1] == 0).all()


def test_attention_f64_semantics():
    """GQA head mapping, K/V broadcast over the batch, softcap and peaked scores, on a case small enough to state by hand."""
    from oracle.oracle import attention_f64
    rng = np.random.default_rng(3)
    q = rng.standard_normal((2, 4, 3, 32)).astype(np.float32)
    k = rng.standard_normal((1, 2, 5, 32)).astype(np.float16)
    v = rng.standard_normal((1, 2, 5, 32)).astype(np.float16)
    got = attention_f64(q, k, v, None, 0.3, 0.0)
    for b in range(2):
        for h in range(4):
            s = 0.3 * q[b, h].astype(np.float16).astype(np.float64) @ k[0, h // 2].astype(np.float64).T
            p = np.exp(s - s.max(-1, keepdims=True))
            assert np.allclose(got[b, :, h], (p / p.sum(-1, keepdims=True)) @ v[0, h // 2].astype(np.float64), rtol=0, atol=1e-12)
    capped = attention_f64(q * 100, k, v, None, 0.3, 5.0)
    s = 5.0 * np.tanh(float(np.float32(0.3) / np.float32(5.0)) * (q[0, 0] * 100).astype(np.float16).astype(np.float64) @ k[0, 0].astype(np.float64).T)
    p = np.exp(s - s.max(-1, keepdims=True))
    assert np.allclose(capped[0, :, 0], (p / p.sum(-1, keepdims=True)) @ v[0, 0].astype(np.float64), rtol=0, atol=1e-12)


@pytest.mark.parametrize("kw,pos", [
    (dict(n_dims=128, mode=0), [0, 1, 7, 4095, 100000]),
    (dict(n_dims=128, mode=2), [0, 3, 100000]),
    (dict(n_dims=64, mode=0), [5, 77777]),                                            # dims 64..127 pass through
    (dict(n_dims=64, mode=2, with_ff=True, freq_base=500000.0), [9, 100000]),         # freq_factors (Llama 3)
    (dict(n_dims=128, mode=0, ext_factor=1.0, freq_scale=0.25, n_ctx_orig=4096, attn_factor=1.0), [0, 5, 300]),   # YaRN ramp + mscale
    (dict(n_dims=128, mode=2, ext_factor=0.5, freq_scale=0.5, n_ctx_orig=2048, beta_fast=16.0, beta_slow=2.0), [1, 60]),
])
def test_rope_ref_matches_ggml_cpu_rope(ref, kw, pos):
    """rope_ref against ggml_rope_ext on the reference's CPU backend: within 8 f32 ulps of |x0| + |x1| of each pair (times
    mscale).  (YaRN at large positions is left out: where the ramp mixes the two thetas, ggml's f32 expression may be
    contracted into an FMA, which moves theta by an ulp -- 1e-2 rad at pos 1e5.)"""
    from oracle.oracle import rope_ref
    kw = dict(kw)
    rng = np.random.default_rng(len(pos) + kw["n_dims"])
    if kw.pop("with_ff", False):
        kw["freq_factors"] = rng.uniform(1.0, 8.0, kw["n_dims"] // 2).astype(np.float32)
    x = rng.standard_normal((len(pos), 6, 128)).astype(np.float32)
    p = np.array(pos, dtype=np.int32)
    want = ref.rope_ext(x, p, **kw)
    got = rope_ref(x, p, **kw)
    nd = kw["n_dims"]
    pair = np.abs(x).copy()
    if kw["mode"] == 0:
        pair[..., 0:nd:2] = pair[..., 1:nd:2] = np.abs(x[..., 0:nd:2]) + np.abs(x[..., 1:nd:2])
    else:
        pair[..., :nd // 2] = pair[..., nd // 2:nd] = np.abs(x[..., :nd // 2]) + np.abs(x[..., nd // 2:nd])
    mscale = 1.0 + (0.1 * np.log(1.0 / kw["freq_scale"]) if kw.get("ext_factor", 0.0) else 0.0)
    bound = 8 * 2.0 ** -24 * pair * mscale * kw.get("attn_factor", 1.0)
    err = np.abs(got - want)
    assert (err <= bound).all(), float((err / bound).max())
    assert np.array_equal(got[..., nd:], x[..., nd:].astype(np.float64))
    if pos[0] == 0 and not kw.get("ext_factor"):
        assert np.array_equal(got[0], x[0].astype(np.float64))   # pos 0: ROPE is exactly the identity

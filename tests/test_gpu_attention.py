"""GPU tests (an H100, sm_90a): the attention kernels against the float64 restatement of FLASH_ATTN_EXT
(oracle.attention_f64) and of ROPE (oracle.rope_ref), both pinned to ggml's CPU code in tests/test_oracle.py.

Kernels: the tensor-core prefill kernel (flash_attn_mma.cu, path 2), the scalar kernel (ops.cu, path 1) and the attention
phase of the persistent decode kernel (decode_flow.cu, through b200_attn_program).

Bars, per output element.  A_d = sum_j p_j |v_jd| / sum_j p_j, from the float64 reference.
  eta       u ((D + 4) scale max_j sum_i |q_i k_ji| + 4 softcap + 4 max_j |s_j| + 2 max_j |mask_j|), u = 2^-24: a bound on the
            fp32 error of any one score (the dot product's gamma_D, then the scale, tanh, mask and max-subtraction roundings).
            Relative errors <= eta in every p_j move the output by at most 2 eta A_d.
  fp32 kernels (scalar, decode)   |err| <= (C32 + 2 eta) A_d
  tensor-core kernel              |err| <= (2^-11 + C32 + 2 eta) A_d + 2^-25 sum_j |v_jd| / sum_j p_j
            P is rounded to f16 for the P.V MMA: relative 2^-11 where it is a normal f16, absolute 2^-25 where it is subnormal;
            the denominator sums the unrounded P.
  C32       exp, the fp32 accumulation over the keys and the final division.
  Rows whose keys are all masked must be exactly 0; every output must be finite.
"""
import numpy as np
import pytest
import torch

from oracle.oracle import Q4_K, Q5_K, Q6_K, attention_f64, random_blocks, rope_ref

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DEV = "cuda"
C32 = 1e-5
F16 = np.float16
WORST = {}


@pytest.fixture(scope="module")
def host():
    import llama_cpp_b200.host as h
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test without a GPU")
    assert h.device_count() >= 1, "libb200qmm.so sees no sm_90 device"
    yield h
    for name, r in sorted(WORST.items()):
        print(f"worst err/bound over the module, {name}: {r:.3f}")


def bound_terms(q, k, v, mask, scale, softcap):
    """eta [B, N, H, 1] and S_d = sum_j |v_jd| / sum_j p_j [B, N, H, DV] over the live keys, same layouts as attention_f64."""
    B, H, N, D = q.shape
    Bk, Hkv, n_kv, _ = k.shape
    DV = v.shape[3]
    sc = float(np.float32(scale) / np.float32(softcap)) if softcap else float(scale)
    eta = np.zeros((B, N, H, 1))
    S = np.zeros((B, N, H, DV))
    q16 = q.astype(F16).astype(np.float64)
    g = H // Hkv
    for b in range(B):
        for hk in range(Hkv):
            kk = k[b // (B // Bk), hk].astype(np.float64)
            vv = np.abs(v[b // (B // v.shape[0]), hk].astype(np.float64))
            hs = slice(hk * g, (hk + 1) * g)
            dots = q16[b, hs] @ kk.T
            qk = np.abs(q16[b, hs]) @ np.abs(kk).T
            s = dots * sc
            if softcap:
                s = softcap * np.tanh(s)
            m = np.zeros_like(s)
            if mask is not None:
                m = np.stack([mask[b % mask.shape[0], h % mask.shape[1], :N, :n_kv] for h in range(hk * g, (hk + 1) * g)]).astype(np.float64)
            live = m != -np.inf
            s = np.where(live, s + np.where(live, m, 0.0), -np.inf)
            smax = s.max(-1, keepdims=True)
            p = np.where(live, np.exp(s - np.where(np.isfinite(smax), smax, 0.0)), 0.0)
            l = p.sum(-1, keepdims=True)
            lm = lambda x: np.where(live, x, 0.0).max(-1, keepdims=True)
            e = U * ((D + 4) * scale * lm(qk) + 4 * softcap + 4 * lm(np.abs(np.where(live, s, 0.0))) + 2 * lm(np.abs(m)))
            eta[b, :, hs] = e.transpose(1, 0, 2)
            S[b, :, hs] = ((live.astype(np.float64) @ vv) / np.where(l > 0, l, 1.0)).transpose(1, 0, 2)
    return eta, S


def check(name, got, want, A, eta, S=None, extra=None):
    """got / want / A [..., DV]; eta [..., 1]; S: the tensor-core kernel's subnormal-P term; extra: an additional relative term."""
    assert np.isfinite(got).all(), f"{name}: non-finite output"
    rel = C32 + 2 * eta + (extra if extra is not None else 0.0) + (2.0 ** -11 if S is not None else 0.0)
    bound = rel * A + (2.0 ** -25 * S if S is not None else 0.0)
    err = np.abs(got.astype(np.float64) - want)
    dead = A == 0
    assert (got[dead] == 0).all(), f"{name}: a fully masked row is not exactly 0"
    ok = err <= bound
    ratio = float((err[~dead] / bound[~dead]).max()) if (~dead).any() else 0.0
    kernel = name.split(" ")[0]
    WORST[kernel] = max(WORST.get(kernel, 0.0), ratio)
    print(f"{name}: worst err/bound {ratio:.3f}")
    if not ok.all():
        i = np.unravel_index(np.argmax(np.where(ok, 0, err / np.where(bound > 0, bound, 1))), err.shape)
        raise AssertionError(f"{name}: err {err[i]:.3e} > bound {bound[i]:.3e} at {i} (got {got[i]}, want {want[i]}); "
                             f"{int((~ok).sum())} of {ok.size} elements over")


# ------------------------------------------------------------------------------------------------ prefill (FLASH_ATTN_EXT)
def causal(N, n_kv):
    """query i sits at position n_kv - N + i and sees keys j <= that (llama's causal mask for a prompt at the end of the cache)."""
    return np.arange(n_kv)[None, :] <= (n_kv - N + np.arange(N))[:, None]


def make_mask(rng, kind, N, n_kv, H, B):
    """[m3, m2, N, n_kv] f16 and the cells masked for every row (whose K/V may hold garbage), or (None, None)."""
    if kind == "none":
        return None, None
    allowed = causal(N, n_kv)[None, None]
    dead_cols = np.zeros(n_kv, bool)
    vals = np.zeros((1, 1, N, n_kv))
    if kind == "holes":                                      # other sequences' cells: -inf in every row
        dead_cols = rng.random(n_kv) < 0.15
        allowed = allowed & ~dead_cols
    elif kind == "per_head":
        allowed = allowed & (rng.random((1, H, N, n_kv)) > 0.2)
    elif kind == "finite":                                   # no -inf at all, a different plane per batch
        allowed = np.ones((B, 1, N, n_kv), bool)
        vals = rng.uniform(-3, 3, (B, 1, N, n_kv))
    elif kind == "full":                                     # whole rows and a whole 64 x 64 tile masked
        allowed = np.broadcast_to(allowed, (1, 1, N, n_kv)).copy()
        allowed[..., [1, N // 2], :] = False
        allowed[..., :64, 64:128] = False
    m = np.where(allowed, vals, -np.inf).astype(F16)
    return m, dead_cols


def run_prefill(host, rng, path, D, N, n_kv, H, Hkv, B=2, kind="causal", softcap=0.0, q_mul=1.0, unaligned=False, rows=None, check_flags=True):
    """q as llama's permuted view of Qcur [B, N, H, D]; K/V views of a cache [n_cells, Hkv, D] with every kv head in one row,
    broadcast over the batch; cells past n_kv hold NaN (never read), cells masked in every row hold +-60000 (must not matter).
    Returns the device result [B, N, H, D]."""
    dev = DEV
    qs = (rng.standard_normal((B, N, H, D)) * q_mul).astype(np.float32)
    n_cells = n_kv + 5
    kc = rng.standard_normal((n_cells, Hkv, D)).astype(F16)
    vc = rng.standard_normal((n_cells, Hkv, D)).astype(F16)
    kc[n_kv:] = np.nan
    vc[n_kv:] = np.nan
    mask, dead = make_mask(rng, kind, N, n_kv, H, B)
    if dead is not None and dead.any():
        kc[:n_kv][dead] = rng.choice([-60000.0, 60000.0], size=(int(dead.sum()), Hkv, D)).astype(F16)
        vc[:n_kv][dead] = rng.choice([-60000.0, 60000.0], size=(int(dead.sum()), Hkv, D)).astype(F16)
    q_t = torch.from_numpy(qs).to(dev).permute(0, 2, 1, 3)                        # [B, H, N, D], nb1 = H * D * 4
    kc_t, vc_t = torch.from_numpy(kc).to(dev), torch.from_numpy(vc).to(dev)
    k_t = kc_t[:n_kv].permute(1, 0, 2).unsqueeze(0)                                # [1, Hkv, n_kv, D]
    v_t = vc_t[:n_kv].permute(1, 0, 2).unsqueeze(0)
    m_t = None
    if mask is not None:
        # rows past N hold NaN (never read); unaligned: a row pitch that is not a multiple of 16 bytes and a base 2 bytes off
        pitch = n_kv if not unaligned else n_kv + (5 if (n_kv + 5) % 8 else 6)
        buf = np.full(mask.shape[:2] + (N + 3, pitch + (1 if unaligned else 0)), np.nan, F16)
        off = 1 if unaligned else 0
        buf[:, :, :N, off:off + n_kv] = mask
        m_t = torch.from_numpy(buf).to(dev)[:, :, :, off:off + n_kv]
    scale = 1.0 / np.sqrt(D)
    dst = torch.full((B, N, H, D), float("nan"), dtype=torch.float32, device=dev)
    ws = None
    if path != 1:
        nws = host.flash_attn_workspace_bytes(q_t, k_t, m_t)
        ws = torch.empty(max(nws, 1), dtype=torch.uint8, device=dev)
    host.flash_attn(q_t, k_t, v_t, m_t, dst, scale, softcap, ws=ws, path=path)
    got = dst.cpu().numpy()
    if path == 2 and check_flags:
        dst2 = torch.full_like(dst, float("nan"))
        host.flash_attn(q_t, k_t, v_t, m_t, dst2, scale, softcap, ws=None, path=2)
        assert np.array_equal(got.view(np.uint32), dst2.cpu().numpy().view(np.uint32)), "tile pre-pass changes the result"
    sel = slice(None) if rows is None else rows
    q_ref = np.ascontiguousarray(qs.transpose(0, 2, 1, 3)[:, :, sel])
    k_ref = np.ascontiguousarray(kc[:n_kv].transpose(1, 0, 2))[None]
    v_ref = np.ascontiguousarray(vc[:n_kv].transpose(1, 0, 2))[None]
    m_ref = None if mask is None else np.ascontiguousarray(mask[:, :, sel])
    want, A = attention_f64(q_ref, k_ref, v_ref, m_ref, scale, softcap, want_abs=True)
    eta, S = bound_terms(q_ref, k_ref, v_ref, m_ref, scale, softcap)
    name = f"{'mma' if path == 2 else 'scalar' if path == 1 else 'auto'} D={D} N={N} n_kv={n_kv} H={H}/{Hkv} B={B} mask={kind}" + \
           (" unaligned" if unaligned else "") + (f" softcap={softcap}" if softcap else "") + (f" q*{q_mul}" if q_mul != 1 else "")
    check(name, got[:, sel], want, A, eta, S if path == 2 else None)
    return got


@pytest.mark.parametrize("D", [64, 128])
def test_mma_ragged_shapes(host, D):
    """Every (N, n_kv) pair of ragged q-tiles and kv tail tiles, causal, GQA 4, K/V broadcast over two sequences."""
    rng = np.random.default_rng(D)
    for N in (16, 17, 63, 64, 65, 200):
        for n_kv in (1, 63, 64, 65, 1000, 1001, 4097):
            run_prefill(host, rng, 2, D, N, n_kv, 8, 2, kind="causal")


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("kind,gqa,unaligned", [
    ("none", 1, False), ("causal", 4, False), ("holes", 8, False), ("per_head", 4, False), ("finite", 1, False),
    ("causal", 8, True), ("holes", 4, True), ("full", 1, False), ("full", 8, True),
])
def test_mma_masks(host, D, kind, gqa, unaligned):
    rng = np.random.default_rng(D * 1000 + sum(map(ord, kind)) * 10 + gqa + 5 * unaligned)
    for N, n_kv in ((65, 1001), (200, 4097), (17, 130)):
        run_prefill(host, rng, 2, D, N, n_kv, 8, 8 // gqa, kind=kind, unaligned=unaligned)


@pytest.mark.parametrize("D", [64, 128])
def test_mma_softcap_and_peaked_scores(host, D):
    rng = np.random.default_rng(7 + D)
    run_prefill(host, rng, 2, D, 65, 1001, 8, 2, kind="causal", softcap=30.0)
    run_prefill(host, rng, 2, D, 64, 300, 4, 4, kind="holes", softcap=50.0, q_mul=20.0)
    run_prefill(host, rng, 2, D, 200, 1000, 8, 1, kind="holes", q_mul=20.0)           # |s| ~ 50
    run_prefill(host, rng, 2, D, 33, 4097, 8, 8, kind="full", q_mul=20.0)


def test_mma_benchmarked_shape(host):
    """pp2048 of Llama-3-8B: N = n_kv = 2048, 32 heads over 8 kv heads, D = 128, causal; the whole output is computed on the
    device and rows {0, 1, 63, 64, 1023, 2047} plus 40 random rows of every head are checked."""
    rng = np.random.default_rng(2048)
    rows = np.unique(np.concatenate([[0, 1, 63, 64, 1023, 2047], rng.choice(2048, 40, replace=False)]))
    got = run_prefill(host, rng, 2, 128, 2048, 2048, 32, 8, B=1, kind="causal", rows=rows)
    assert np.isfinite(got).all()


def test_auto_path_is_one_of_the_two_kernels(host):
    """path 0 (what the backend runs) is bit-identical to the tensor-core kernel from 16 rows on, and to the scalar kernel below."""
    for N, want_path in ((15, 1), (16, 2), (100, 2)):
        outs = []
        for path in (0, want_path):
            outs.append(run_prefill(host, np.random.default_rng(N), path, 128, N, 333, 8, 2, kind="holes", check_flags=False))
        assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), N


@pytest.mark.parametrize("D", [32, 64, 96, 128, 256])
def test_scalar_kernel(host, D):
    """The scalar kernel (every decode step on the per-op path, prefill below 16 rows): N in {1, 2, 7, 15} and 64 forced, the
    same GQA / mask / softcap cases as the tensor-core kernel."""
    rng = np.random.default_rng(300 + D)
    cases = [(1, 1, "none", 1, 0.0), (2, 65, "causal", 4, 0.0), (7, 1001, "holes", 8, 0.0), (15, 300, "per_head", 4, 0.0),
             (64, 1001, "full", 1, 0.0), (7, 200, "finite", 8, 30.0), (15, 4097, "causal", 4, 0.0), (2, 130, "holes", 1, 50.0)]
    for N, n_kv, kind, gqa, softcap in cases:
        run_prefill(host, rng, 1, D, N, n_kv, 8, 8 // gqa, kind=kind, softcap=softcap)
    run_prefill(host, rng, 1, D, 1, 1000, 8, 2, kind="holes", q_mul=20.0)


# ------------------------------------------------------------------------------------------------ decode attention phase
D_HEAD = 128


def part_range(n_kv, nsplit, part):
    """The keys part `part` of a split head walks (decode_flow.cu, attn_phase: chunks rounded up to 32 keys)."""
    chunk = ((n_kv + nsplit - 1) // nsplit + 31) // 32 * 32
    return min(n_kv, part * chunk), min(n_kv, (part + 1) * chunk)


def f16_ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(F16)).astype(np.float64)


def run_decode(host, rng, n_head, Hkv, n_kv, kpos, mask_kind="none", softcap=0.0, rope=None, pos=0, masked_part=None, nsplit_known=None,
               qkv=None):
    """One launch of b200_attn_program; checks the cache writes and the output.  Returns (nsplit, output)."""
    dev = DEV
    D = D_HEAD
    rope = dict(rope or {})
    ff = rope.pop("freq_factors", None)
    n_cells = n_kv + 9
    kc = rng.standard_normal((n_cells, Hkv, D)).astype(F16)
    vc = rng.standard_normal((n_cells, Hkv, D)).astype(F16)
    kc[n_kv:] = np.nan                                        # never read
    vc[n_kv:] = np.nan
    kc[kpos] = np.nan                                         # the new token's cell: the phase must use its own k / v
    vc[kpos] = np.nan
    mask = None
    if mask_kind != "none":
        mask = rng.uniform(-2, 0, n_kv)
        if mask_kind == "pad":                                # llama pads n_kv: cells past the last used one are -inf
            mask[max(kpos + 1, n_kv - 37):] = -np.inf
        elif mask_kind == "holes":
            mask[rng.random(n_kv) < 0.2] = -np.inf
        elif mask_kind == "part":                             # every key of one split part
            k0, k1 = part_range(n_kv, nsplit_known, masked_part)
            mask[k0:k1] = -np.inf
        mask[kpos] = 0.0
        dead = mask == -np.inf
        dead[kpos] = False
        kc[:n_kv][dead] = rng.choice([-60000.0, 60000.0], size=(int(dead.sum()), Hkv, D)).astype(F16)
        vc[:n_kv][dead] = rng.choice([-60000.0, 60000.0], size=(int(dead.sum()), Hkv, D)).astype(F16)
        mask = mask.astype(F16)
    q = rng.standard_normal(n_head * D).astype(np.float32)
    k = rng.standard_normal(Hkv * D).astype(np.float32)
    v = rng.standard_normal(Hkv * D).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    q_t, k_t, v_t = T(q), T(k), T(v)
    kc_t, vc_t = T(kc), T(vc)
    dst = torch.full((n_head * D,), float("nan"), dtype=torch.float32, device=dev)
    scale = 1.0 / np.sqrt(D)
    kw = dict(n_dims=rope.get("n_dims", D), rope_mode=rope.get("mode", 0), freq_base=rope.get("freq_base", 10000.0),
              freq_scale=rope.get("freq_scale", 1.0), ext_factor=rope.get("ext_factor", 0.0), attn_factor=rope.get("attn_factor", 1.0),
              beta_fast=rope.get("beta_fast", 32.0), beta_slow=rope.get("beta_slow", 1.0), n_ctx_orig=rope.get("n_ctx_orig", 0))
    qkv_dev = None
    if qkv is not None:
        qkv_dev = dict(qkv)
        q_t.fill_(float("nan")); k_t.fill_(float("nan")); v_t.fill_(float("nan"))
    nsplit = host.attn_program(q_t, k_t, v_t, dst, kc_t, vc_t, T(np.array([kpos], np.int64)), T(np.array([kpos], np.int64)),
                               T(np.array([pos], np.int32)), n_head, Hkv, n_kv, scale, softcap, mask=None if mask is None else T(mask),
                               freq_factors=None if ff is None else T(np.asarray(ff, np.float32)), qkv=qkv_dev, **kw)
    if DEV == "cuda":
        torch.cuda.synchronize()
    if qkv is not None:                                       # teacher forcing: the mat-vec phase's own q / k / v
        q, k, v = q_t.cpu().numpy(), k_t.cpu().numpy(), v_t.cpu().numpy()
        assert np.isfinite(q).all() and np.isfinite(k).all() and np.isfinite(v).all()
    got = dst.cpu().numpy()
    kc2, vc2 = kc_t.cpu().numpy(), vc_t.cpu().numpy()
    # ---- cache writes: row kpos of every kv head = f16(ROPE(k)) within one f16 ulp plus the fp32 ROPE error; v exactly; nothing else
    rk = rope_ref(k.reshape(1, Hkv, D), np.array([pos], np.int32), kw["n_dims"], kw["rope_mode"], kw["freq_base"], kw["freq_scale"],
                  kw["ext_factor"], kw["attn_factor"], kw["beta_fast"], kw["beta_slow"], kw["n_ctx_orig"], ff)[0]
    rq = rope_ref(q.reshape(1, n_head, D), np.array([pos], np.int32), kw["n_dims"], kw["rope_mode"], kw["freq_base"], kw["freq_scale"],
                  kw["ext_factor"], kw["attn_factor"], kw["beta_fast"], kw["beta_slow"], kw["n_ctx_orig"], ff)[0]
    mscale = kw["attn_factor"] * (1.0 + 0.1 * np.log(1.0 / kw["freq_scale"]) if kw["ext_factor"] else 1.0)

    def rope_err(x):                                          # 8 f32 ulps of |x0| + |x1| of each rotated pair (times mscale)
        x = np.abs(x.reshape(-1, D)).astype(np.float64)
        nd = kw["n_dims"]
        e = np.zeros_like(x)
        a, b = (slice(0, nd, 2), slice(1, nd, 2)) if kw["rope_mode"] == 0 else (slice(0, nd // 2), slice(nd // 2, nd))
        e[:, a] = e[:, b] = 8 * U * (x[:, a] + x[:, b]) * mscale
        return e

    want_k16 = rk.astype(F16).astype(np.float64)
    krow = kc2[kpos].astype(np.float64)
    kerr = np.abs(krow - want_k16)
    assert (kerr <= np.maximum(f16_ulp(want_k16), f16_ulp(krow)) + rope_err(k)).all(), f"k cache row: max err {kerr.max()}"
    assert np.array_equal(vc2[kpos].view(np.uint16), v.reshape(Hkv, D).astype(F16).view(np.uint16)), "v cache row != f16(v)"
    others = np.arange(n_cells) != kpos
    assert np.array_equal(kc2[others].view(np.uint16), kc[others].view(np.uint16)), "k cache written outside row kpos"
    assert np.array_equal(vc2[others].view(np.uint16), vc[others].view(np.uint16)), "v cache written outside row kpos"
    # ---- output: against attention_f64 over the cache the kernel wrote
    k_ref = np.ascontiguousarray(kc2[:n_kv].transpose(1, 0, 2))[None]
    v_ref = np.ascontiguousarray(vc2[:n_kv].transpose(1, 0, 2))[None]
    q_ref = rq.reshape(1, n_head, 1, D)
    m_ref = None if mask is None else mask.reshape(1, 1, 1, n_kv)
    want, A = attention_f64(q_ref, k_ref, v_ref, m_ref, scale, softcap, want_abs=True)
    eta, _ = bound_terms(q_ref, k_ref, v_ref, m_ref, scale, softcap)
    extra = None
    if pos != 0 or kw["ext_factor"]:
        # the kernel's f16 q may differ from f16(rope_ref(q)) by one f16 ulp plus the fp32 ROPE error, element by element:
        # that moves score j by at most scale sum_i dq_i |k_ji| and the output by twice that (relative) times A_d
        dq = f16_ulp(rq.reshape(n_head, D)) + rope_err(q)
        g = n_head // Hkv
        kabs = np.abs(k_ref[0].astype(np.float64))
        live = np.ones(n_kv, bool) if mask is None else mask != -np.inf
        ds = np.stack([(dq[h] @ kabs[h // g].T)[live].max() for h in range(n_head)]) * scale
        extra = (2 * ds).reshape(1, 1, n_head, 1)
    name = f"decode H={n_head}/{Hkv} n_kv={n_kv} nsplit={nsplit} kpos={kpos} mask={mask_kind}" + (f" softcap={softcap}" if softcap else "") + \
           (f" pos={pos} rope={rope}" if pos or rope else "") + (" +qkv" if qkv is not None else "")
    check(name, got.reshape(1, 1, n_head, D), want, A, eta, extra=extra)
    return nsplit, got


def test_decode_split_coverage(host):
    """n_head in {8, 32, 128} (several, about 4 and 1 CTAs per head on an H100) x n_kv from 1 to 9000: single-part heads,
    2-, 4- and >= 7-part heads, parts that walk more than one 896-key score tile; kpos at 0, the last key, the middle and a part
    boundary; masks none / padding / holes / one whole part masked."""
    rng = np.random.default_rng(9000)
    seen, multi_tile = set(), False
    for n_head, gqas in ((8, (1, 8)), (32, (4, 1)), (128, (8, 1))):
        for i, n_kv in enumerate((1, 31, 512, 513, 1000, 2049, 4096, 9000)):
            Hkv = n_head // gqas[i % 2]
            kpos = (n_kv - 1, 0, n_kv // 2)[i % 3]
            kind = ("none", "pad", "holes")[i % 3]
            nsplit, _ = run_decode(host, rng, n_head, Hkv, n_kv, kpos, kind, softcap=30.0 if i == 5 else 0.0)
            seen.add(nsplit)
            k0, k1 = part_range(n_kv, nsplit, 0)
            multi_tile |= k1 - k0 > 896
            if nsplit > 1:
                b0, _ = part_range(n_kv, nsplit, 1)
                run_decode(host, rng, n_head, Hkv, n_kv, b0, "holes")            # kpos: first key of part 1
                run_decode(host, rng, n_head, Hkv, n_kv, b0 - 1, "none")         # ... last key of part 0
                run_decode(host, rng, n_head, Hkv, n_kv, n_kv - 1, "part", masked_part=0, nsplit_known=nsplit)
                run_decode(host, rng, n_head, Hkv, n_kv, 0, "part", masked_part=1, nsplit_known=nsplit)
    print(f"nsplit values seen: {sorted(seen)}; a part walked more than 896 keys: {multi_tile}")
    assert {1, 2, 4} <= seen and max(seen) >= 7, sorted(seen)
    assert multi_tile


@pytest.mark.parametrize("rope,pos", [
    (dict(mode=0), 100000),
    (dict(mode=2), 77777),
    (dict(mode=0, n_dims=64), 4321),
    (dict(mode=2, n_dims=64), 100000),
    (dict(mode=2, freq_base=500000.0, freq_factors=np.linspace(1.0, 8.0, 64)), 100000),
    (dict(mode=0, ext_factor=1.0, freq_scale=0.25, n_ctx_orig=4096), 300),    # YaRN: ramp mix and mscale
    (dict(mode=2, ext_factor=1.0, freq_scale=0.25, n_ctx_orig=4096, beta_fast=16.0, beta_slow=2.0), 37),
])
def test_decode_rope(host, rope, pos):
    """ROPE fused into the phase: mode 0 and NEOX, n_dims < head_dim, freq_factors, YaRN, positions up to 100000."""
    rng = np.random.default_rng(pos)
    run_decode(host, rng, 32, 8, 1000, 999, "holes", rope=rope, pos=pos)
    run_decode(host, rng, 8, 1, 300, 17, "none", rope=rope, pos=pos)


@pytest.mark.parametrize("n_head,Hkv,n_kv", [(32, 8, 300), (32, 8, 2049), (8, 2, 300), (8, 2, 2049)])
def test_decode_from_tagged_slots(host, n_head, Hkv, n_kv):
    """q | k | v produced by the fused mat-vec phase of the same launch (the production case), read through tagged slots;
    the reference is teacher-forced with the q / k / v the phase also wrote to its plain buffers."""
    rng = np.random.default_rng(n_head * n_kv)
    n_embd = 4096
    types = (Q4_K, Q6_K, Q5_K)
    rows = (n_head * D_HEAD, Hkv * D_HEAD, Hkv * D_HEAD)
    ws = [host.to_device_weights(random_blocks(t, m, n_embd, rng)) for t, m in zip(types, rows)]
    x = torch.from_numpy(rng.standard_normal(n_embd).astype(np.float32)).to(DEV)
    norm_w = torch.from_numpy(rng.uniform(0.5, 1.5, n_embd).astype(np.float32)).to(DEV)
    run_decode(host, rng, n_head, Hkv, n_kv, n_kv - 1, "pad", qkv=dict(types=types, ws=ws, x=x, norm_w=norm_w, eps=1e-5))


def test_decode_is_deterministic(host):
    """Three launches of the same split program give bit-identical outputs."""
    outs = [run_decode(host, np.random.default_rng(5), 32, 8, 2049, 2048, "holes")[1] for _ in range(3)]
    assert all(np.array_equal(outs[0].view(np.uint32), o.view(np.uint32)) for o in outs[1:])

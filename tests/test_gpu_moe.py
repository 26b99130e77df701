"""MUL_MAT_ID on an H100 (sm_90a), kernel by kernel, against the oracle (oracle.mul_mat_id, itself pinned to ggml_mul_mat_id on the
reference's CPU backend in test_oracle.py).  The entry points are those of include/b200_moe.h: b200_mul_mat_id_path picks the kernel,
b200_moe_route runs the grouped GEMM's router alone.

Bounds, per output element, with S = sum_k |w_k x_k| (the dequantised weight times the f32 activation):
  router (moe_route_kernel)         exact: every invariant of the tile layout below, against a numpy restatement
  grouped GEMM (path 2)             |gpu - oracle| <= 6e-6 S.  The arithmetic of the plain prefill GEMM (test_gemm_tcgen05_matches_oracle):
                                    the Q8_K integers are the CPU's, the block sums come from fp16-integer MMAs accumulated in fp32, and
                                    only the fp32 combine of the blocks differs from the CPU's order
  grouped GEMM vs plain GEMM        bit-identical: both run gemm_q_wgmma_kernel with the same pre-pass and per-column d_a, and an MMA
                                    column does not depend on where it sits in the tile
  routed GEMV (path 1)              |gpu - oracle| <= 4e-6 S, the bar of every GEMV test (integer dot products, fp32 order only)
  repeated launches                 bit-identical, although the router's atomics place the columns differently each time; permuting the
                                    tokens permutes the output bit-exactly
Activations are N(0, 1) unless a case says otherwise; every case has one all-zero 256-block and one all-zero activation column.  The
output buffer starts as NaN between guard words: every element must be written, nothing outside it.
The worst err / bound of each kernel is printed at the end of the module (pytest -s)."""
import numpy as np
import pytest
import torch

from oracle.oracle import Q4_0, Q4_K, Q5_K, Q6_K, Q8_0, TYPE_NAMES, constant_sign_blocks, random_blocks, saturated_blocks

pytestmark = pytest.mark.gpu

NT = 128                                   # columns per tile of the grouped GEMM
WORST = {}                                 # kernel -> worst err / bound seen


@pytest.fixture(scope="module")
def host():
    import llama_cpp_b200.host as h
    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test without a GPU")
    assert h.device_count() >= 1, "libb200qmm.so sees no sm_90 device"
    yield h
    for k, v in sorted(WORST.items()):
        print(f"MUL_MAT_ID worst err/bound  {k:<28} {v:.3f}")


def note(kernel, ratio):
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(ratio))


# ---------------------------------------------------------------------------------------------------------------- helpers
def strided_ids(ids: np.ndarray, n_expert: int, strided: bool) -> torch.Tensor:
    """ids int32 [T, n_used] on the device; strided: as llama passes them, the first n_used columns of an [T, n_expert] argsort."""
    T, n_used = ids.shape
    if not strided:
        return torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int32)).cuda()
    full = np.tile(np.arange(n_expert, dtype=np.int32)[::-1], (T, 1))   # the columns past n_used: ids no kernel may read
    full[:, :n_used] = ids
    v = torch.from_numpy(full).cuda()[:, :n_used]
    assert v.stride(0) == n_expert
    return v


def top_k_ids(rng, T, E, n_used):
    return np.stack([rng.permutation(E)[:n_used] for _ in range(T)]).astype(np.int32)


def device_experts(host, w: np.ndarray) -> torch.Tensor:
    E, M, rb = w.shape
    return host.to_device_weights(w.reshape(E * M, rb)).view(E, M, rb)


def abs_scale(oracle, t, w, b, ids) -> np.ndarray:
    """S = sum_k |w_k x_k| of every output, f64 [T, n_used, M]."""
    E, M, _ = w.shape
    T, nb1, K = b.shape
    n_used = ids.shape[1]
    out = np.zeros((T, n_used, M))
    cols = np.abs(b[:, np.arange(n_used) % nb1].astype(np.float64))                      # [T, n_used, K]
    for e in np.unique(ids):
        deq = np.abs(np.stack([oracle.dequantize(t, w[e, m], K) for m in range(M)]).astype(np.float64))
        sel = ids == e
        out[sel] = cols[sel] @ deq.T
    return out


def guarded(T, n_used, M, G=64):
    """A NaN-filled [T, n_used, M] output with G guard words on each side: (full buffer, the output view)."""
    n = T * n_used * M
    full = torch.full((n + 2 * G,), float("nan"), device="cuda")
    full[:G] = -1234.5
    full[n + G:] = -1234.5
    return full, full[G:G + n].view(T, n_used, M)


def check_guarded(full, G=64):
    f = full.cpu().numpy()
    assert (f[:G] == -1234.5).all() and (f[-G:] == -1234.5).all(), "write outside dst"
    assert np.isfinite(f[G:-G]).all(), f"{int((~np.isfinite(f[G:-G])).sum())} outputs not written"
    return f[G:-G]


def run_checked(host, oracle, t, w, b, ids, path, kernel, strided=False, E=None, want_taken=None):
    """path 0/1/2 through b200_mul_mat_id_path into a guarded NaN buffer; checks every element against the oracle."""
    E = E or w.shape[0]
    T, nb1, K = b.shape
    n_used, M = ids.shape[1], w.shape[1]
    full, out = guarded(T, n_used, M)
    _, taken = host.mul_mat_id(t, device_experts(host, w), torch.from_numpy(b).cuda(), strided_ids(ids, E, strided), path=path, out=out)
    torch.cuda.synchronize()
    assert taken == (want_taken or path), taken
    got = check_guarded(full).reshape(T, n_used, M)
    want = oracle.mul_mat_id(t, w, b, ids)
    bound = (6e-6 if taken == 2 else 4e-6) * abs_scale(oracle, t, w, b, ids) + 1e-30
    err = np.abs(got - want)
    ratio = float((err / bound).max())
    note(kernel, ratio)
    assert (err <= bound).all(), (TYPE_NAMES[t], kernel, float(err.max()), ratio)
    return got


def with_zero_blocks(b):
    b[0, 0, :256] = 0.0                    # a zero activation block
    b[min(1, b.shape[0] - 1)] = 0.0        # an all-zero column (every slot of token 1)
    return b


# ---------------------------------------------------------------------------------------------------------------- router
def route_ids_counts(rng, counts, n_used=1):
    """ids [T, n_used] giving expert e exactly counts[e] jobs, in random order."""
    jobs = np.concatenate([np.full(c, e, np.int32) for e, c in enumerate(counts)])
    rng.shuffle(jobs)
    assert jobs.size % n_used == 0
    return jobs.reshape(-1, n_used)


def check_route(ids, n_expert, nb1, te, cs, cd):
    """The tile layout moe_route_kernel must produce, restated."""
    T, n_used = ids.shape
    R = T * n_used
    max_tiles = -(-R // NT) + n_expert
    assert te.shape == (max_tiles,) and cs.shape == (max_tiles, NT) and cd.shape == (max_tiles, NT)
    flat = ids.reshape(-1)
    cnt = np.bincount(flat, minlength=n_expert)
    ntile = -(-cnt // NT)
    live = int(ntile.sum())
    # experts in ascending order, each with a contiguous run of ceil(cnt / 128) tiles; -1 past the live tiles
    assert np.array_equal(te[:live], np.repeat(np.arange(n_expert), ntile))
    assert (te[live:] == -1).all()
    cs, cd = cs.reshape(-1), cd.reshape(-1)
    assert (cs[live * NT:] == -1).all() and (cd[live * NT:] == -1).all()
    base = 0
    for e in range(n_expert):
        run_d, run_s = cd[base * NT:(base + ntile[e]) * NT], cs[base * NT:(base + ntile[e]) * NT]
        c = cnt[e]
        assert (run_d[:c] >= 0).all() and (flat[run_d[:c]] == e).all(), e      # the first cnt_e slots: this expert's jobs
        assert (run_d[c:] == -1).all() and (run_s[c:] == -1).all(), e          # the rest of the run: padding
        base += ntile[e]
    used = cd[cd >= 0]
    assert np.array_equal(np.sort(used), np.arange(R))                          # every job exactly once
    pos = np.nonzero(cd >= 0)[0]
    t, s = cd[pos] // n_used, cd[pos] % n_used
    assert np.array_equal(cs[pos], t * nb1 + (s if nb1 > 1 else 0))
    assert (cs[cd < 0] == -1).all()


ROUTE_CASES = {
    "uniform": dict(E=8, n_used=2, T=300, nb1=2, strided=False),
    "one_expert": dict(E=8, n_used=2, T=200, nb1=1, strided=True, ids="one"),
    "counts_0_1_127_128_129": dict(E=6, n_used=1, T=None, nb1=1, strided=False, ids="counts"),
    "counts_strided": dict(E=6, n_used=1, T=None, nb1=1, strided=True, ids="counts"),
    "E1": dict(E=1, n_used=1, T=130, nb1=1, strided=False),
    "E60_k4": dict(E=60, n_used=4, T=97, nb1=4, strided=True),
    "E256_k8": dict(E=256, n_used=8, T=70, nb1=1, strided=True),
    "repeated_in_row": dict(E=8, n_used=4, T=50, nb1=4, strided=True, ids="repeat"),
}


@pytest.mark.parametrize("case", sorted(ROUTE_CASES))
def test_router_invariants(host, case):
    c = ROUTE_CASES[case]
    rng = np.random.default_rng(sorted(ROUTE_CASES).index(case))
    E, n_used = c["E"], c["n_used"]
    kind = c.get("ids")
    if kind == "counts":
        ids = route_ids_counts(rng, [0, 1, 127, 128, 129, 300])
    elif kind == "one":
        ids = np.full((c["T"], n_used), 5, np.int32)
    elif kind == "repeat":
        ids = rng.integers(0, E, size=(c["T"], n_used)).astype(np.int32)
        ids[::3, 1] = ids[::3, 0]
        ids[7] = 2
    else:
        ids = top_k_ids(rng, c["T"], E, n_used)
    nb1 = c["nb1"] if c["nb1"] == 1 else n_used
    te, cs, cd = host.moe_route(strided_ids(ids, max(E, n_used), c["strided"]), E, nb1)
    torch.cuda.synchronize()
    check_route(ids, E, nb1, te.cpu().numpy(), cs.cpu().numpy(), cd.cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------- grouped GEMM
GROUPED_CASES = {
    # name: (type, E, n_used, M, K, T, nb1 == 1, strided ids, ids kind)
    "q4K_ragged_M200_K2304": (Q4_K, 8, 2, 200, 2304, 80, True, True, "topk"),
    "q5K_M96_K256": (Q5_K, 8, 2, 96, 256, 100, False, False, "topk"),
    "q6K_ragged_M200_K2304": (Q6_K, 8, 2, 200, 2304, 64, False, True, "topk"),
    "q4K_tile_edges": (Q4_K, 6, 1, 130, 512, None, True, False, "counts"),
    "q6K_tile_edges_strided": (Q6_K, 6, 1, 64, 256, None, True, True, "counts"),
    "q6K_E60_k4": (Q6_K, 60, 4, 64, 512, 40, False, True, "topk"),
    "q5K_E256_k8": (Q5_K, 256, 8, 64, 256, 40, True, True, "topk"),
    "q4K_repeated_in_row": (Q4_K, 8, 2, 128, 256, 48, False, False, "repeat"),
}


@pytest.mark.parametrize("case", sorted(GROUPED_CASES))
def test_grouped_gemm_matches_oracle(host, oracle, case):
    t, E, n_used, M, K, T, nb1_one, strided, kind = GROUPED_CASES[case]
    rng = np.random.default_rng(100 + sorted(GROUPED_CASES).index(case))
    if kind == "counts":
        ids = route_ids_counts(rng, [0, 1, 127, 128, 129, 40])
        T = ids.shape[0]
    elif kind == "repeat":
        ids = top_k_ids(rng, T, E, n_used)
        ids[::2, 1] = ids[::2, 0]
    else:
        ids = top_k_ids(rng, T, E, n_used)
    nb1 = 1 if nb1_one else n_used
    w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
    b = with_zero_blocks(rng.standard_normal((T, nb1, K)).astype(np.float32))
    run_checked(host, oracle, t, w, b, ids, 2, "grouped GEMM", strided=strided)


@pytest.mark.parametrize("t", [Q4_K, Q5_K, Q6_K])
def test_grouped_gemm_saturated_blocks(host, oracle, t):
    """Every weight field at its extreme and every Q8_K integer +-127 (oracle.saturated_blocks): a block's integer sum is above 2^24,
    beyond what fp32 holds exactly, and the MMA accumulates it in fp32.  Same bound as everywhere else."""
    rng = np.random.default_rng(700 + t)
    E, n_used, M, K, T = 4, 2, 160, 2304, 96
    w = np.stack([saturated_blocks(t, M, K, rng) for _ in range(E)])
    b = constant_sign_blocks(T * n_used, K, rng).reshape(T, n_used, K)
    ids = top_k_ids(rng, T, E, n_used)
    run_checked(host, oracle, t, w, b, ids, 2, f"grouped GEMM saturated {TYPE_NAMES[t]}")


# ---------------------------------------------------------------------------------------------------------------- Mixtral-8x7B shapes
MIXTRAL = {
    "ffn_gate_q4K": (Q4_K, 14336, 4096, True),         # gate / up: one activation column per token (nb1 = 1)
    "ffn_down_q6K": (Q6_K, 4096, 14336, False),        # down: one column per (token, slot) (nb1 = n_used)
}
_mixtral_cache = {}


def mixtral_case(host, name):
    """E = 8, n_used = 2, T = 512 (a pp512 prompt): weights, activations, llama-strided top-2 ids and the grouped GEMM's output."""
    if name not in _mixtral_cache:
        _mixtral_cache.clear()
        t, M, K, nb1_one = MIXTRAL[name]
        E, n_used, T = 8, 2, 512
        rng = np.random.default_rng(51 + M % 1000)
        w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
        nb1 = 1 if nb1_one else n_used
        b = with_zero_blocks(rng.standard_normal((T, nb1, K)).astype(np.float32))
        ids = top_k_ids(rng, T, E, n_used)
        wd = device_experts(host, w)
        bd = torch.from_numpy(b).cuda()
        full, out = guarded(T, n_used, M)
        _, taken = host.mul_mat_id(t, wd, bd, strided_ids(ids, E, True), path=0, out=out)
        torch.cuda.synchronize()
        assert taken == 2                                      # what the backend runs for a Mixtral prompt
        got = check_guarded(full).reshape(T, n_used, M)
        _mixtral_cache[name] = (t, w, wd, b, bd, ids, got)
    return _mixtral_cache[name]


@pytest.mark.parametrize("name", sorted(MIXTRAL))
def test_mixtral_shapes_sampled_rows(host, oracle, name):
    """48 weight rows of every expert, every token, against oracle.mul_mat_id(t, w[:, rows], b, ids): a row's dot product does not depend
    on the other rows, so the oracle on the sub-problem is its answer for those elements (test_bench_shapes_sampled_rows_and_columns)."""
    t, w, wd, b, bd, ids, got = mixtral_case(host, name)
    M = w.shape[1]
    rng = np.random.default_rng(9)
    rows = np.unique(np.concatenate([[0, 1, 127, 128, M - 1], rng.integers(0, M, size=43)]))
    ws = np.ascontiguousarray(w[:, rows])
    want = oracle.mul_mat_id(t, ws, b, ids)
    err = np.abs(got[:, :, rows] - want)
    bound = 6e-6 * abs_scale(oracle, t, ws, b, ids) + 1e-30
    ratio = float((err / bound).max())
    note("grouped GEMM (Mixtral)", ratio)
    assert (err <= bound).all(), (name, float(err.max()), ratio)


@pytest.mark.parametrize("name", sorted(MIXTRAL))
def test_grouped_gemm_bit_identical_to_plain_gemm(host, name):
    """Each expert's columns gathered and run through the plain prefill GEMM (b200_mul_mat, path 2) on that expert's weights, at full size."""
    t, w, wd, b, bd, ids, got = mixtral_case(host, name)
    T, nb1, K = b.shape
    n_used = ids.shape[1]
    host.lib().b200_set_mul_mat_path(2)
    try:
        for e in range(w.shape[0]):
            tok, slot = np.nonzero(ids == e)
            x = bd[torch.from_numpy(tok).cuda(), torch.from_numpy(slot % nb1).cuda()].contiguous()      # [n_e, K]
            y = host.mul_mat(t, wd[e], x).cpu().numpy()
            same = y.view(np.uint32) == got[tok, slot].view(np.uint32)
            assert same.all(), (name, e, int((~same).sum()), float(np.abs(y - got[tok, slot]).max()))
    finally:
        host.lib().b200_set_mul_mat_path(0)


# ---------------------------------------------------------------------------------------------------------------- determinism
@pytest.mark.parametrize("nb1_one", [True, False])
def test_grouped_gemm_deterministic_and_token_permutation(host, nb1_one):
    rng = np.random.default_rng(61 + nb1_one)
    t, E, n_used, M, K, T = Q4_K, 8, 2, 256, 1024, 300
    w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
    nb1 = 1 if nb1_one else n_used
    b = rng.standard_normal((T, nb1, K)).astype(np.float32)
    ids = top_k_ids(rng, T, E, n_used)
    wd = device_experts(host, w)
    runs = [host.mul_mat_id(t, wd, torch.from_numpy(b).cuda(), strided_ids(ids, E, True), path=2)[0].cpu().numpy() for _ in range(3)]
    for r in runs[1:]:
        assert np.array_equal(r.view(np.uint32), runs[0].view(np.uint32))
    perm = rng.permutation(T)
    y, taken = host.mul_mat_id(t, wd, torch.from_numpy(np.ascontiguousarray(b[perm])).cuda(), strided_ids(ids[perm], E, True), path=2)
    assert taken == 2
    assert np.array_equal(y.cpu().numpy().view(np.uint32), runs[0][perm].view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------- routed GEMV
@pytest.mark.parametrize("nb1_one", [True, False])
@pytest.mark.parametrize("t", [Q4_0, Q8_0, Q4_K, Q5_K, Q6_K])
def test_routed_gemv_matches_oracle(host, oracle, t, nb1_one):
    rng = np.random.default_rng(200 + t + 50 * nb1_one)
    E, n_used, M, K, T = 8, 2, 72, 512, 12
    w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
    nb1 = 1 if nb1_one else n_used
    b = with_zero_blocks(rng.standard_normal((T, nb1, K)).astype(np.float32))
    ids = top_k_ids(rng, T, E, n_used)
    ids[3] = [5, 5]                                              # the same expert twice
    run_checked(host, oracle, t, w, b, ids, 1, "routed GEMV", strided=True)


def test_routed_gemv_token_chunks(host, oracle):
    """n_used = 8, T = 8200: 65600 (token, slot) rows, more than gridDim.y takes, so the GEMV runs in chunks of 65535 / 8 = 8191 tokens.
    Sampled tokens on both sides of the chunk edge, against the oracle; every output written."""
    rng = np.random.default_rng(8191)
    t, E, n_used, M, K, T = Q4_K, 8, 8, 32, 256, 8200
    w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
    b = rng.standard_normal((T, 1, K)).astype(np.float32)
    ids = top_k_ids(rng, T, E, n_used)
    full, out = guarded(T, n_used, M)
    _, taken = host.mul_mat_id(t, device_experts(host, w), torch.from_numpy(b).cuda(), strided_ids(ids, E, True), path=1, out=out)
    torch.cuda.synchronize()
    assert taken == 1
    got = check_guarded(full).reshape(T, n_used, M)
    toks = np.unique(np.concatenate([[0, 1, 8189, 8190, 8191, 8192, 8193, T - 1], rng.integers(0, T, size=24)]))
    want = oracle.mul_mat_id(t, w, b[toks], ids[toks])
    bound = 4e-6 * abs_scale(oracle, t, w, b[toks], ids[toks]) + 1e-30
    err = np.abs(got[toks] - want)
    note("routed GEMV", float((err / bound).max()))
    assert (err <= bound).all(), (float(err.max()), float((err / bound).max()))


# ---------------------------------------------------------------------------------------------------------------- dispatch
@pytest.mark.parametrize("t,T,n_used,E,want", [
    (Q4_K, 16, 2, 8, 2),                   # T * n_used = 32: the grouped GEMM
    (Q6_K, 31, 1, 8, 1),                   # 31: the GEMV
    (Q4_0, 64, 2, 8, 1),                   # Q4_0 / Q8_0 experts have no grouped GEMM
    (Q8_0, 64, 2, 8, 1),
    (Q4_K, 32, 2, 257, 1),                 # more experts than the router's shared counters
])
def test_dispatch(host, oracle, t, T, n_used, E, want):
    rng = np.random.default_rng(T * E + t)
    M, K = 40, 512
    w = np.stack([random_blocks(t, M, K, rng) for _ in range(E)])
    b = rng.standard_normal((T, 1, K)).astype(np.float32)
    ids = top_k_ids(rng, T, E, n_used)
    run_checked(host, oracle, t, w, b, ids, 0, "grouped GEMM" if want == 2 else "routed GEMV", strided=True, want_taken=want)
    if want == 1 and T * n_used >= 32:
        with pytest.raises(host.B200Error, match=r"\(-6\)"):
            host.mul_mat_id(t, device_experts(host, w), torch.from_numpy(b).cuda(), strided_ids(ids, E, True), path=2)

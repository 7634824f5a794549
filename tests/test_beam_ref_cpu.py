"""The fp64 statement of st5_beam_topk's scores and the rank checker of tests/beam_contract_ref.py, without a GPU: the
bound holds against an fp32 emulation of the kernel's steps on adversarial rows, it is tight enough that a wrong token
or row is far outside it at the shapes of tests/test_beam_contract_gpu.py, and the checker rejects wrong lists."""
import math

import pytest
import torch

import beam_contract_ref as BR

INF = math.inf


def _rows(kind, BK, V, dtype, g):
    if kind == "grid":      # 1/8 grid: exact ties inside every row
        x = torch.randint(-32, 33, (BK, V), generator=g).float() / 8
    elif kind == "wide":    # logits over +-90 (exp underflows for most of the row)
        x = torch.randn(BK, V, generator=g) * 30
    elif kind == "near":    # a cluster of values one ulp apart near the top
        x = torch.randn(BK, V, generator=g)
        top = torch.full((BK, 16), 5.0)
        x[:, :16] = top + torch.arange(16) * 2.0 ** -21
    else:
        raise ValueError(kind)
    return x.to(dtype)


def _top(sc, K, V, t):
    """The kernel's selection on fp32 scores [BK, V]: per sentence, (score desc, flat asc), first n."""
    BK = sc.shape[0]
    B = BK // K
    flat = sc.view(B, K, V)[:, 0] if t == 0 else sc.reshape(B, K * V)
    n = min(2 * K, flat.shape[1] - 1)
    v, i = torch.sort(flat.double(), dim=1, descending=True, stable=True)
    return v[:, :n].float(), i[:, :n] % V, i[:, :n] // V


@pytest.mark.parametrize("kind", ["grid", "wide", "near"])
@pytest.mark.parametrize("V", [81, 8000, 32768])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("fma", [False, True])
def test_bound_holds_against_fp32_emulation(kind, V, dtype, fma):
    K, B, eos = 2, 2, 2
    g = torch.Generator().manual_seed(V + len(kind))
    x = _rows(kind, B * K, V, dtype, g)
    cum = -torch.rand(B * K, generator=g) * 300
    mask = torch.zeros(V)
    mask[1], mask[5] = -INF, -0.75
    worst = 0.0
    for it in (0.5, 1.0, 1.25):
        for t, mn, mx in ((0, 1, 50), (4, 1, 50), (4, 9, 50)):
            z, b = BR.scores(x, cum, mask, it, eos, t, mn, mx, K)
            e = BR.emulate(x, cum, mask, it, eos, t, mn, mx, fma=fma)
            e = e.view(B, K, V)[:, 0] if t == 0 else e.reshape(B, K * V)
            assert torch.equal(e == -INF, z == -INF)
            f = torch.isfinite(z)
            r = ((e.double() - z).abs()[f] / b[f]).max()
            assert r <= 1.0, (it, t, float(r))
            worst = max(worst, float(r))
    assert worst > 1e-3  # (the bound is within three orders of magnitude of what fp32 really does)


def test_bound_is_not_vacuous_at_the_gpu_shapes():
    """At the GPU test's logits (1/8 grid and N(0, 9), cum down to -4, V up to 32768) the bound is far below the
    score change of one wrong token on the grid (1/16 at inv_temp 0.5) or of one wrong row's cum."""
    g = torch.Generator().manual_seed(0)
    for V in (81, 8000, 32768):
        K = 2
        x = torch.cat([_rows("grid", 1, V, torch.float32, g), torch.randn(1, V, generator=g) * 3])
        cum = -torch.rand(K, generator=g) * 4
        for t in (0, 5):
            _, b = BR.scores(x, cum, torch.zeros(V), 1.25, 2, t, 1, 50, K)
            assert float(b.max()) < 2e-5, (V, t, float(b.max()))
            assert float(b.max()) < (1 / 16) / 1000


def _lists(K, V, t, g, dtype=torch.float32, tie_rows=True):
    B = 2
    x = torch.randint(-16, 17, (B * K, V), generator=g).float().div(8).to(dtype)
    cum = -torch.rand(B * K, generator=g) * 3
    if tie_rows:  # sentence 0: rows 0 and K - 1 identical (logits and cum), their tokens 10 and 11 on top
        x[0, 10:12] = 6.0
        x[K - 1], cum[K - 1] = x[0], cum[0]
    mask = torch.zeros(V)
    mask[1] = -INF
    e = BR.emulate(x, cum, mask, 1.0, 2, t, 1, 50)
    sc, tk, bm = _top(e, K, V, t)
    z, b = BR.scores(x, cum, mask, 1.0, 2, t, 1, 50, K)
    return x, cum, mask, z, b, sc, tk, bm


def _check(x, cum, mask, z, b, sc, tk, bm, K, V, t, s=0):
    same = BR.same_inputs(x, cum, mask, 2, K, s, t)
    return BR.check_sentence(z[s], b[s], sc[s], tk[s], bm[s], V, same, what="planted")


@pytest.mark.parametrize("K,V,t", [(1, 81, 0), (4, 81, 3), (5, 9, 3), (16, 81, 7), (16, 3, 2), (3, 5, 0)])
def test_checker_accepts_the_emulated_selection(K, V, t):
    g = torch.Generator().manual_seed(K * 100 + V)
    args = _lists(K, V, t, g)
    for s in range(2):
        assert _check(*args, K, V, t, s=s) <= 1.0


def test_checker_rejects_planted_wrong_lists():
    K, V, t = 4, 81, 3
    g = torch.Generator().manual_seed(5)
    x, cum, mask, z, b, sc, tk, bm = _lists(K, V, t, g)
    _check(x, cum, mask, z, b, sc, tk, bm, K, V, t)
    n = sc.shape[1]

    def bad(sc2, tk2, bm2, match):
        with pytest.raises(AssertionError, match=match):
            _check(x, cum, mask, z, b, sc2, tk2, bm2, K, V, t)

    # a swapped pair (two well separated picks exchanged, scores with them)
    gap = (z[0].sort(descending=True).values[:n].diff().abs() > 1e-3).nonzero().flatten()
    i = int(gap[0])
    p = list(range(n))
    p[i], p[i + 1] = i + 1, i
    bad(sc[:, p], tk[:, p], bm[:, p], "descending|ranked after")
    # a swapped pair of tokens only: each score is off its own pair's
    tk2 = tk.clone()
    tk2[0, i], tk2[0, i + 1] = tk[0, i + 1], tk[0, i]
    bm2 = bm.clone()
    bm2[0, i], bm2[0, i + 1] = bm[0, i + 1], bm[0, i]
    if not (torch.equal(tk2, tk) and torch.equal(bm2, bm)):
        bad(sc, tk2, bm2, "off its own pair")
    # a duplicate
    tk2, bm2, sc2 = tk.clone(), bm.clone(), sc.clone()
    tk2[0, 3], bm2[0, 3], sc2[0, 3] = tk[0, 2], bm[0, 2], sc[0, 2]
    bad(sc2, tk2, bm2, "picked twice")
    # the best candidate missing (the list shifted up, the (n+1)-th appended)
    e = BR.emulate(x, cum, mask, 1.0, 2, t, 1, 50)
    v, ii = torch.sort(e.reshape(2, K * V).double(), dim=1, descending=True, stable=True)
    sc2 = torch.cat([sc[:, 1:], v[:, n:n + 1].float()], 1)
    tk2 = torch.cat([tk[:, 1:], ii[:, n:n + 1] % V], 1)
    bm2 = torch.cat([bm[:, 1:], ii[:, n:n + 1] // V], 1)
    bad(sc2, tk2, bm2, "left out|within bound")


def test_checker_rejects_ties_in_the_wrong_order():
    K, V, t = 4, 81, 3
    g = torch.Generator().manual_seed(11)
    x, cum, mask, z, b, sc, tk, bm = _lists(K, V, t, g)
    # within a row: two picks of one beam with bit-identical logits
    row = [(i, j) for i in range(sc.shape[1]) for j in range(i + 1, sc.shape[1])
           if bm[0, i] == bm[0, j] and sc[0, i] == sc[0, j]]
    # across beams: rows 0 and K - 1 are identical, so their copies of a token tie
    cross = [(i, j) for i in range(sc.shape[1]) for j in range(i + 1, sc.shape[1])
             if bm[0, i] != bm[0, j] and tk[0, i] == tk[0, j] and sc[0, i] == sc[0, j]]
    assert row and cross
    for i, j in (row[0], cross[0]):
        p = list(range(sc.shape[1]))
        p[i], p[j] = j, i
        with pytest.raises(AssertionError, match="tie"):
            _check(x, cum, mask, z, b, sc[:, p], tk[:, p], bm[:, p], K, V, t)
    # the tie at the cut: the last pick replaced by an identical candidate of higher flat index
    n = sc.shape[1]
    zf = z[0]
    last = int(bm[0, n - 1]) * V + int(tk[0, n - 1])
    same = BR.same_inputs(x, cum, mask, 2, K, 0, t)
    picked = set((bm[0] * V + tk[0]).tolist())
    cand = [c for c in torch.nonzero(zf == zf[last]).flatten().tolist()
            if c > last and c not in picked and bool(same(last, torch.tensor([c]))[0])]
    if cand:
        tk2, bm2 = tk.clone(), bm.clone()
        tk2[0, n - 1], bm2[0, n - 1] = cand[0] % V, cand[0] // V
        with pytest.raises(AssertionError, match="tie"):
            _check(x, cum, mask, z, b, sc, tk2, bm2, K, V, t)


def test_all_minus_inf_sentence_picks_the_lowest_flat_indices():
    K, V, t = 3, 5, 4
    x = torch.full((2 * K, V), -INF)
    cum = torch.zeros(2 * K)
    mask = torch.zeros(V)
    z, b = BR.scores(x, cum, mask, 1.0, 2, t, 1, 50, K)
    n = min(2 * K, K * V - 1)
    f = torch.arange(n)
    sc = torch.full((n,), -INF)
    BR.check_sentence(z[0], b[0], sc, f % V, f // V, V)
    with pytest.raises(AssertionError, match="tie"):
        f2 = f.clone()
        f2[-1] = n
        BR.check_sentence(z[0], b[0], sc, f2 % V, f2 // V, V)

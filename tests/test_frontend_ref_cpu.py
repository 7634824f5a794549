"""The fp64 statements of tests/frontend_ref.py (layer 0 of the waveform extractor) and of the decode attention in
tests/attention_ref.py checked on their own (no GPU): against independent statements (fp64 autograd through F.conv1d,
nn.GroupNorm, F.layer_norm and F.gelu; layer 0 of the oracle's ConvFeatureExtractionModel in both modes;
attention_ref.forward and a plain torch.softmax), and by showing that each of a list of one-line kernel defects, put
into the statement, leaves the bound the GPU test uses at that test's shapes."""
import math
import os
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import attention_ref as A
import frontend_ref as R

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.speecht5_oracle_asr import ConvFeatureExtractionModel  # noqa: E402

F64 = torch.float64
EPS = 1e-5
SMS = 132  # H100 SXM; the GPU test reads the count from the device
TORCH_GELU = {"gelu": "none", "gelu_tanh": "tanh"}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _case(B, C, K, S, T0, seed=0, kind="rand"):
    g = _gen(seed)
    n = (T0 - 1) * S + K
    if kind == "rand":
        wave = torch.randn(B, n, generator=g, dtype=F64) * 0.1
    elif kind == "const":
        wave = torch.full((B, n), 0.3, dtype=F64)
    else:
        wave = torch.zeros(B, n, dtype=F64)
    wave = wave.float().double()
    w = (torch.randn(C, K, generator=g, dtype=F64) / math.sqrt(K)).float().double()
    gamma = (1.0 + 0.2 * torch.randn(C, generator=g, dtype=F64)).float().double()
    beta = (0.2 * torch.randn(C, generator=g, dtype=F64)).float().double()
    dy = torch.randn(B, T0, C, generator=g, dtype=F64)
    return wave, w, gamma, beta, dy


def _autograd(mode, wave, w, gamma, beta, dy, S, approximate):
    """y [B, T0, C] and the gradients of sum(y * dy) wrt w, gamma, beta, in fp64 through torch's modules."""
    w, gamma, beta = (t.clone().requires_grad_(True) for t in (w, gamma, beta))
    v = F.conv1d(wave[:, None], w[:, None], stride=S)                      # [B, C, T0]
    if mode == "gn":
        gn = nn.GroupNorm(w.shape[0], w.shape[0], eps=EPS).double()
        with torch.no_grad():
            gn.weight.copy_(gamma)
            gn.bias.copy_(beta)
        z = F.group_norm(v, w.shape[0], gamma, beta, EPS).transpose(1, 2)
        assert torch.allclose(gn(v).transpose(1, 2), z, rtol=0, atol=1e-12)
    else:
        z = F.layer_norm(v.transpose(1, 2), (w.shape[0],), gamma, beta, EPS)
    y = F.gelu(z, approximate=approximate)
    (y * dy).sum().backward()
    return y.detach(), w.grad, gamma.grad, beta.grad


def _close(a, b, tol=1e-9):
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


# ============================================================================================ statements vs torch
@pytest.mark.parametrize("mode", ["gn", "ln"])
@pytest.mark.parametrize("act", ["gelu", "gelu_tanh"])
@pytest.mark.parametrize("K,S,T0", [(10, 5, 129), (1, 1, 7), (16, 96, 3), (11, 3, 1)])
def test_statement_matches_fp64_autograd(mode, act, K, S, T0):
    C = 66
    wave, w, gamma, beta, dy = _case(2, C, K, S, T0, seed=K + T0)
    fwd, bwd = (R.gn_forward, R.gn_backward) if mode == "gn" else (R.ln_forward, R.ln_backward)
    f = fwd(wave, w, gamma, beta, S=S, eps=EPS, act=act)
    y, dw, dg, db = _autograd(mode, wave, w, gamma, beta, dy, S, "none")
    _close(f["y"], y)                               # act() states the erf GELU that ST5_ACT_GELU_TANH stands in for
    b = bwd(dy, wave, w, gamma, beta, f["mean"], f["rstd"], S=S, act=act)
    _, dw, dg, db = _autograd(mode, wave, w, gamma, beta, dy, S, TORCH_GELU[act])  # act_grad: the form computed
    _close(b["dw"], dw)
    _close(b["dgamma"], dg)
    _close(b["dbeta"], db)


@pytest.mark.parametrize("mode", ["default", "layer_norm"])
def test_statement_matches_the_oracle_layer0(mode):
    C, K, S = 64, 10, 5
    torch.manual_seed(0)
    m = ConvFeatureExtractionModel([(C, K, S)], mode=mode).double()
    norm = m.conv_layers[0][2]
    with torch.no_grad():
        norm.weight.copy_(1.0 + 0.2 * torch.randn(C, dtype=F64))
        norm.bias.copy_(0.2 * torch.randn(C, dtype=F64))
    wave = torch.randn(3, 5 * 200 + 5, dtype=F64) * 0.1
    y = m(wave).transpose(1, 2).detach()
    w = m.conv_layers[0][0].weight.detach()[:, 0]
    fwd = R.gn_forward if mode == "default" else R.ln_forward
    f = fwd(wave, w, norm.weight.detach(), norm.bias.detach(), S=S, eps=norm.eps, act="gelu")
    assert f["y"].shape == y.shape
    _close(f["y"], y)


def test_frames_and_taps():
    assert R.frames(9, 10, 5) == 0 and R.frames(10, 10, 5) == 1 and R.frames(14, 10, 5) == 1
    assert R.frames(15, 10, 5) == 2 and R.frames(160000, 10, 5) == 31999
    wave = torch.arange(2 * 23, dtype=F64).view(2, 23)
    x = R.taps(wave, 4, 6)                                                  # T0 = 4; samples 22 unused
    assert x.shape == (2, 4, 4) and float(x[1, 3, 3]) == 23 + 3 * 6 + 3


def test_decode_statement_matches_attention_forward_and_softmax():
    B, H, Tk = 3, 4, 150
    q, k, v, _ = A.make_inputs(B, H, 1, Tk, seed=3, dtype=torch.float32)
    kp = torch.zeros(B, Tk, dtype=torch.uint8)
    kp[1, 64:128] = 1
    kp[2, 5:] = 1
    f = A.decode_forward(q[:, :, 0], k, v, scale=0.125, key_pad=kp)
    g = A.forward(q, k, v, scale=0.125, key_pad=kp)
    assert torch.equal(f["out"], g["out"]) and torch.equal(f["P"], g["P"])
    s = 0.125 * torch.einsum("bhc,bhjc->bhj", q.double()[:, :, 0], k.double())
    s = s.masked_fill(kp.bool()[:, None], -math.inf)
    p = torch.softmax(s, -1)
    _close(f["P"][:, :, 0], p, 1e-14)
    _close(f["out"][:, :, 0], torch.einsum("bhj,bhjc->bhc", p, v.double()), 1e-14)


def test_decode_all_masked_rows_are_zero():
    q, k, v, _ = A.make_inputs(2, 2, 1, 70, seed=4, dtype=torch.float32)
    kp = torch.zeros(2, 70, dtype=torch.uint8)
    kp[1] = 1
    f = A.decode_forward(q[:, :, 0], k, v, scale=0.125, key_pad=kp)
    b = A.decode_bounds(f, u=2.0 ** -24)
    assert bool((f["out"][1] == 0).all()) and bool((f["P"][1] == 0).all())
    assert bool((b["out"][1] <= A.TINY).all()) and bool(torch.isfinite(f["out"][0]).all())


# ============================================================================================ defects leave the bound
def _gn(B=3, C=64, K=10, S=5, T0=129, seed=1, kind="rand", u=R.R.U32, act="gelu"):
    wave, w, gamma, beta, dy = _case(B, C, K, S, T0, seed=seed, kind=kind)
    f = R.gn_forward(wave, w, gamma, beta, S=S, eps=EPS, act=act)
    return f, R.gn_forward_bounds(f, u), (wave, w, gamma, beta, dy)


def _rstd(var):
    return 1.0 / torch.sqrt(var + EPS)


@pytest.mark.parametrize("T0", [127, 129, 385])
def test_gn_variance_over_t0_minus_1_leaves_bound(T0):
    f, b, _ = _gn(T0=T0)
    assert R.exceeds(_rstd(f["var"] * T0 / (T0 - 1)), f["rstd"], b["rstd"])


@pytest.mark.parametrize("T0", [129, 385, 300])
def test_gn_last_partial_chunk_losing_a_frame_leaves_bound(T0):
    f, b, _ = _gn(T0=T0)
    v = f["v"][:, :-1]
    mean = v.mean(1)
    var = ((v - mean[:, None]) ** 2).mean(1)
    assert R.exceeds(mean, f["mean"], b["mean"]) or R.exceeds(_rstd(var), f["rstd"], b["rstd"])


def test_gn_pilot_counted_twice_leaves_bound():
    f, b, _ = _gn(T0=300)
    T0 = 300
    pilots = f["v"][:, ::R.TCH].sum(1)
    assert R.exceeds((f["v"].sum(1) + pilots) / T0, f["mean"], b["mean"])


@pytest.mark.parametrize("kind", ["const", "silence"])
def test_gn_eps_outside_the_sqrt_leaves_bound(kind):
    f, b, _ = _gn(C=96, T0=300, kind=kind)
    assert R.exceeds(1.0 / (torch.sqrt(f["var"]) + EPS), f["rstd"], b["rstd"])


def _gn_bwd(**kw):
    f, _, (wave, w, gamma, beta, dy) = _gn(**kw)
    mean, rstd = f["mean"].float().double(), f["rstd"].float().double()
    S = kw.get("S", 5)
    bw = R.gn_backward(dy, wave, w, gamma, beta, mean, rstd, S=S, act="gelu")
    C, K = w.shape
    z = [torch.ones(C, K, dtype=F64), torch.ones(C, dtype=F64), torch.ones(C, dtype=F64)]
    return bw, R.gn_backward_bounds(bw, *z), z, (wave, w, S)


def test_gn_dgamma_dbeta_swapped_leaves_bound():
    bw, bb, (dw0, dg0, db0), _ = _gn_bwd()
    assert R.exceeds(dg0 + bw["dbeta"], dg0 + bw["dgamma"], bb["dgamma"])
    assert R.exceeds(db0 + bw["dgamma"], db0 + bw["dbeta"], bb["dbeta"])


def test_gn_dv_without_the_xhat_m2_term_leaves_bound():
    bw, bb, (dw0, _, _), _ = _gn_bwd()
    dv = bw["rstd"] * bw["gamma"] * (bw["g"] - bw["m1"])
    assert R.exceeds(dw0 + torch.einsum("btc,btk->ck", dv, bw["x"]), dw0 + bw["dw"], bb["dw"])


@pytest.mark.parametrize("K,S", [(10, 5), (2, 1), (16, 96)])
def test_gn_dw_tap_shifted_by_one_sample_leaves_bound(K, S):
    bw, bb, (dw0, _, _), (wave, w, S_) = _gn_bwd(C=33, K=K, S=S, T0=130)
    x1 = R.taps(torch.cat([wave, torch.zeros(wave.shape[0], 1, dtype=F64)], 1)[:, 1:], K, S)   # sample t S + k + 1
    bad = bw["dw"].clone()
    bad[:, K - 1] = torch.einsum("btc,bt->c", bw["dv"], x1[..., K - 1])
    assert R.exceeds(dw0 + bad, dw0 + bw["dw"], bb["dw"])


def _ln(B=2, C=66, K=10, S=5, T0=150, seed=2, u=R.R.U32, act="gelu"):
    wave, w, gamma, beta, dy = _case(B, C, K, S, T0, seed=seed)
    f = R.ln_forward(wave, w, gamma, beta, S=S, eps=EPS, act=act)
    return f, R.ln_forward_bounds(f, u), (wave, w, gamma, beta, dy)


@pytest.mark.parametrize("C", [2, 66, 512])
def test_ln_odd_channel_using_the_even_gamma_leaves_bound(C):
    f, b, (wave, w, gamma, beta, dy) = _ln(C=C, u=R.R.U_BF16)
    g_bad = gamma.view(-1, 2)[:, :1].expand(-1, 2).reshape(-1)
    assert R.exceeds(R.R.act(f["xhat"] * g_bad + beta, "gelu"), f["y"], b["y"])


def test_ln_variance_over_c_minus_1_leaves_bound():
    f, b, _ = _ln(C=66)
    assert R.exceeds(_rstd(f["var"] * 66 / 65).reshape(-1), f["rstd"].reshape(-1), b["rstd"])


@pytest.mark.parametrize("B,T0", [(2, 90), (3, 5000)])
def test_ln_taps_from_10_dropped_at_k11_leaves_bound(B, T0):
    """The KH = 5 instantiation (taps 0..9) run at K = 11 would leave tap 10 unaccumulated."""
    wave, w, gamma, beta, dy = _case(B, 66, 11, 3, T0, seed=6)
    f = R.ln_forward(wave, w, gamma, beta, S=3, eps=EPS, act="gelu_tanh")
    bw = R.ln_backward(dy, wave, w, gamma, beta, f["mean"].reshape(-1), f["rstd"].reshape(-1), S=3, act="gelu_tanh")
    z = [torch.ones(66, 11, dtype=F64), torch.ones(66, dtype=F64), torch.ones(66, dtype=F64)]
    bb = R.ln_backward_bounds(bw, *z, SMS)
    bad = bw["dw"].clone()
    bad[:, 10] = 0
    assert R.exceeds(z[0] + bad, z[0] + bw["dw"], bb["dw"])


def _dec(B=3, H=12, Tk=129, seed=5, dtype=torch.float32):
    q, k, v, _ = A.make_inputs(B, H, 1, Tk, seed=seed, dtype=dtype)
    q = q[:, :, 0]
    f = A.decode_forward(q, k, v, scale=0.125)
    return (q, k, v), f, A.decode_bounds(f, u=2.0 ** -24 if dtype == torch.float32 else 2.0 ** -8)


@pytest.mark.parametrize("Tk,drop", [(65, 63), (65, 64), (129, 128), (1500, 64), (1500, 1499), (64, 63)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_decode_dropping_a_key_leaves_bound(Tk, drop, dtype):
    (q, k, v), f, b = _dec(Tk=Tk, dtype=dtype)
    kp = torch.zeros(q.shape[0], Tk, dtype=torch.uint8)
    kp[:, drop] = 1
    g = A.decode_forward(q, k, v, scale=0.125, key_pad=kp)
    assert R.exceeds(g["P"][:, :, 0], f["P"][:, :, 0], b["P"])
    if dtype == torch.float32:  # (a bf16 output's rounding can hide one key among 1500)
        assert R.exceeds(g["out"][:, :, 0], f["out"][:, :, 0], b["out"])


def _splits(f, Tk):
    """Per-split (m_s, l_s, acc_s) in fp64, as the split kernel forms them."""
    s = f["s"][:, :, 0]
    v = f["v"]
    out = []
    for j0 in range(0, Tk, A.DCH):
        ss = s[..., j0:j0 + A.DCH]
        m = ss.amax(-1, keepdim=True)
        e = torch.exp(ss - m)
        out.append((m, e.sum(-1, keepdim=True), torch.einsum("bhj,bhjc->bhc", e, v[:, :, j0:j0 + A.DCH])))
    return out


@pytest.mark.parametrize("Tk,bad_split", [(129, 0), (129, 2), (1500, 11)])
def test_decode_merging_a_split_without_its_rescale_leaves_bound(Tk, bad_split):
    (q, k, v), f, b = _dec(Tk=Tk)
    sp = _splits(f, Tk)
    M = torch.stack([m for m, _, _ in sp]).amax(0)
    r = sum(a * (1.0 if i == bad_split else torch.exp(m - M)) for i, (m, _, a) in enumerate(sp))
    L = sum(l * torch.exp(m - M) for m, l, _ in sp)
    assert R.exceeds(r / L, f["out"][:, :, 0], b["out"])


@pytest.mark.parametrize("Tk", [65, 129, 1500])
def test_decode_split_probs_without_1_over_l_leave_bound(Tk):
    (q, k, v), f, b = _dec(Tk=Tk)
    s = f["s"][:, :, 0]
    assert R.exceeds(torch.exp(s - s.amax(-1, keepdim=True)), f["P"][:, :, 0], b["P"])

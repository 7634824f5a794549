"""The fp64 statement of tests/rowops_ref.py checked on its own (no GPU): against independent statements (torch.nn
modules and autograd in fp64, F.pad + slicing, and the reference's own fairseq Adam class), and by showing that each of
a list of one-line kernel defects, put into the statement, leaves the bound the GPU test uses at that test's shapes."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import rowops_ref as R

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader as rl  # noqa: E402

F64 = torch.float64
SEED, OFFSET = 99, 5
SMS = 132  # H100 SXM; the GPU test reads the count from the device
needs_ref = pytest.mark.skipif(not rl.available(), reason="reference tree not available")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ln_case(rows, C, drop=0.1, seed=0, offset=False, const=False):
    g = _gen(seed)
    x = torch.randn(rows, C, generator=g, dtype=F64)
    res = torch.randn(rows, C, generator=g, dtype=F64)
    if offset:
        res += 100.0
    if const:
        x[::3] = 0.0
        res[::3] = 0.7
    gamma = 1.0 + 0.2 * torch.randn(C, generator=g, dtype=F64)
    beta = 0.2 * torch.randn(C, generator=g, dtype=F64)
    kp = R.keep((rows, C), drop, SEED, OFFSET) if drop > 0 else None
    ds = R.D.drop_scale(drop)
    return x, res, gamma, beta, kp, ds


# ============================================================================================ independent statements
@pytest.mark.parametrize("drop", [0.0, 0.1])
def test_layernorm_matches_torch_autograd(drop):
    rows, C = 37, 80
    x, res, gamma, beta, kp, dsc = _ln_case(rows, C, drop)
    xa = x.clone().requires_grad_()
    mask = kp.to(F64) * dsc if kp is not None else 1.0
    s = res + xa * mask
    ln = torch.nn.LayerNorm(C, eps=1e-5, dtype=F64)
    ln.weight.data.copy_(gamma)
    ln.bias.data.copy_(beta)
    y = ln(s)
    dy = torch.randn(rows, C, generator=_gen(3), dtype=F64)
    y.backward(dy)
    f = R.ln_forward(x, gamma, beta, eps=1e-5, residual=res, kp=kp, dscale=dsc)
    assert torch.allclose(f["y"], y.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(f["mean"], s.detach().mean(-1), rtol=1e-12, atol=1e-12)
    b = R.ln_backward(dy, f["s"], f["mean"], f["rstd"], gamma, kp=kp, dscale=dsc)
    assert torch.allclose(b["dx"], xa.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(b["dgamma"], ln.weight.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(b["dbeta"], ln.bias.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(b["dxsum"], xa.grad.sum(0), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("act", ["none", "relu", "tanh"])
@pytest.mark.parametrize("rows", [1, 2, 257])
def test_batchnorm_matches_torch(act, rows):
    C = 37
    g = _gen(rows)
    x = torch.randn(rows, C, generator=g, dtype=F64) * 2 + 0.5
    gamma = 1.0 + 0.3 * torch.randn(C, generator=g, dtype=F64)
    beta = 0.3 * torch.randn(C, generator=g, dtype=F64)
    rm = torch.randn(C, generator=g, dtype=F64)
    rv = torch.rand(C, generator=g, dtype=F64) + 0.5
    drop = 0.1
    kp = R.keep((rows, C), drop, SEED, OFFSET)
    dsc = R.D.drop_scale(drop)
    fn = {"none": lambda t: t, "relu": F.relu, "tanh": torch.tanh}[act]
    for training in (True, False):
        bn = torch.nn.BatchNorm1d(C, eps=1e-5, momentum=0.1, dtype=F64)
        bn.weight.data.copy_(gamma)
        bn.bias.data.copy_(beta)
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
        bn.train(training)
        xa = x.clone().requires_grad_()
        if training and rows == 1:  # torch refuses one value per channel; the kernel uses var = 0 (see the header)
            with pytest.raises(ValueError):
                bn(xa)
            f = R.bn_forward(x, gamma, beta, rm, rv, training=True, momentum=0.1, eps=1e-5, act_name=act)
            assert torch.equal(f["running_var"], 0.9 * rv) and torch.allclose(f["pre"], beta[None])
            continue
        pre = bn(xa)
        y = fn(pre) * kp.to(F64) * dsc
        f = R.bn_forward(x, gamma, beta, rm, rv, training=training, momentum=0.1, eps=1e-5, act_name=act, kp=kp,
                         dscale=dsc)
        assert torch.allclose(f["y"], y.detach(), rtol=1e-10, atol=1e-12)
        if training:
            assert torch.allclose(f["running_mean"], bn.running_mean, rtol=1e-12, atol=1e-14)
            assert torch.allclose(f["running_var"], bn.running_var, rtol=1e-12, atol=1e-14)
        dy = torch.randn(rows, C, generator=_gen(7), dtype=F64)
        y.backward(dy)
        b = R.bn_backward(dy, x, f["pre"], gamma, f["mean"], f["rstd"], act_name=act, kp=kp, dscale=dsc)
        if training:  # (eval: the reference's dx is the batch-statistics form only in training)
            assert torch.allclose(b["dx"], xa.grad, rtol=1e-9, atol=1e-11)
            assert torch.allclose(b["dgamma"], bn.weight.grad, rtol=1e-9, atol=1e-11)
            assert torch.allclose(b["dbeta"], bn.bias.grad, rtol=1e-9, atol=1e-11)


def test_posenc_matches_embedding_autograd():
    B, T, C, V, pad = 3, 11, 16, 9, 1
    g = _gen(4)
    tokens = torch.randint(0, V, (B, T), generator=g)
    tokens[0, :4] = 5  # repeats
    tokens[1, -3:] = pad
    emb = torch.randn(V, C, generator=g, dtype=F64)
    pe = torch.randn(T + 5, C, generator=g, dtype=F64)
    alpha = torch.tensor(1.7, dtype=F64)
    kp = R.keep((B, T, C), 0.1, SEED, OFFSET)
    dsc = R.D.drop_scale(0.1)
    ea, aa = emb.clone().requires_grad_(), alpha.clone().requires_grad_()
    y = (F.embedding(tokens, ea, padding_idx=pad) + aa * pe[:T][None]) * kp.to(F64) * dsc
    dy = torch.randn(B, T, C, generator=g, dtype=F64)
    y.backward(dy)
    yr, _ = R.posenc_forward(pe, 1.7, T, tokens=tokens, emb=emb, kp=kp, dscale=dsc)
    assert torch.allclose(yr, y.detach(), rtol=1e-12, atol=1e-12)
    b = R.posenc_backward(dy, pe, T, tokens=tokens, padding_idx=pad, n_emb=V, kp=kp, dscale=dsc)
    assert torch.allclose(b["demb"], ea.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(b["dalpha"], aa.grad, rtol=1e-12)


@pytest.mark.parametrize("name", ["gelu", "gelu_tanh", "tanh", "relu"])
def test_activation_gradients_match_autograd(name):
    x = torch.cat([torch.linspace(-10, 10, 4001, dtype=F64), torch.zeros(1, dtype=F64)])
    xa = x.clone().requires_grad_()
    fn = {"gelu": F.gelu, "gelu_tanh": lambda t: F.gelu(t, approximate="tanh"), "tanh": torch.tanh,
          "relu": F.relu}[name]
    fn(xa).sum().backward()
    assert torch.allclose(R.act_grad(x, name), xa.grad, rtol=1e-12, atol=1e-14)
    if name != "gelu_tanh":
        assert torch.allclose(R.act(x, name), fn(x), rtol=1e-14, atol=1e-15)
    assert torch.allclose(R.gelu_tanh(x), F.gelu(x, approximate="tanh"), rtol=1e-14, atol=1e-15)
    # the formula part of the GELU_TANH bound
    assert float((R.gelu_tanh(x) - R.gelu(x)).abs().max()) <= R.GELU_TANH_ABS


@pytest.mark.parametrize("d,ph,pad,n_in", [(1, 0, 3, 20), (2, 1, 2, 9), (3, 2, 0, 6), (1, 0, 0, 14)])
def test_lrelu_pad_matches_pad_and_slice(d, ph, pad, n_in):
    B, T, C = 2, 14, 8
    x = torch.randn(B, T, C, generator=_gen(d), dtype=F64)
    slope = 0.1
    lr = F.leaky_relu(x, R.f32(slope))
    padded = F.pad(lr, (0, 0, pad, pad + d * n_in + 4))  # zeros on both sides of the time axis
    want = padded[:, ph::d][:, :n_in]
    assert torch.equal(R.lrelu_pad(x, n_in, d, ph, pad, slope), want)


def _fairseq_adam():
    path = os.path.join(rl.ST5, "fairseq", "fairseq", "optim", "adam.py")
    ns = rl._extract(path, ["Adam"], {"torch": torch, "math": math}, "fairseq.optim.adam")
    return ns["Adam"]


@needs_ref
@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("max_norm", [0.0, 0.5, 1e3])
def test_adam_matches_reference_class(wd, max_norm):
    Adam = _fairseq_adam()
    n = 103
    g0 = _gen(5)
    p = torch.randn(n, generator=g0, dtype=F64)
    lr, b1, b2, eps, gmul = 0.05, 0.9, 0.98, 1e-6, 0.5
    ref_p = torch.nn.Parameter(p.clone())
    opt = Adam([ref_p], lr=R.f32(lr), betas=(R.f32(b1), R.f32(b2)), eps=R.f32(eps), weight_decay=R.f32(wd))
    m = torch.zeros(n, dtype=F64)
    v = torch.zeros(n, dtype=F64)
    cur = p.clone()
    for step in range(1, 6):
        g = torch.randn(n, generator=g0, dtype=F64)
        gn2 = float(R.f32(float((g * g).sum())))
        # fairseq: multiply_grads(grad_mul), then clip_grad_norm_(max_norm) on the scaled gradient
        gs = g * R.f32(gmul)
        if max_norm > 0:
            norm = math.sqrt(gn2) * R.f32(gmul)
            gs = gs * min(R.f32(max_norm) / (norm + 1e-6), 1.0)
        ref_p.grad = gs.clone()
        opt.step()
        out = R.adam_step(cur, g, m, v, lr=lr, beta1=b1, beta2=b2, eps=eps, weight_decay=wd, step=step,
                          grad_norm_sq=gn2, max_norm=max_norm, grad_mul=gmul)
        cur, m, v = out["p"], out["m"], out["v"]
        assert torch.allclose(cur, ref_p.data, rtol=1e-13, atol=1e-15), step
        st = opt.state[ref_p]
        assert torch.allclose(m, st["exp_avg"], rtol=1e-13, atol=1e-15)
        assert torch.allclose(v, st["exp_avg_sq"], rtol=1e-13, atol=1e-15)


def test_adam_skips_on_non_finite_norm():
    p, g, m, v = (torch.randn(9, generator=_gen(i), dtype=F64) for i in range(4))
    v = v.abs()
    for gn2 in (math.nan, math.inf):
        out = R.adam_step(p, g, m, v, lr=1e-3, beta1=0.9, beta2=0.98, eps=1e-6, weight_decay=0.0, step=3,
                          grad_norm_sq=gn2, max_norm=1.0, grad_mul=1.0)
        assert out["skipped"] and torch.equal(out["p"], p) and torch.equal(out["m"], m) and torch.equal(out["v"], v)


# ============================================================================================ defects leave the bound
def test_ln_defects_leave_forward_bounds():
    # variance over C - 1 (C = 8: the GPU test's smallest width)
    x, res, gamma, beta, kp, dsc = _ln_case(64, 8, 0.0)
    f = R.ln_forward(x, gamma, beta, eps=1e-5, residual=res)
    b = R.ln_forward_bounds(f, R.U32)
    C = 8
    rstd_bad = 1.0 / torch.sqrt(f["var"][:, 0] * C / (C - 1) + 1e-5)
    assert R.exceeds(rstd_bad, f["rstd"], b["rstd"])
    # eps outside the square root (constant rows: var = 0), at C = 768 bf16 with the large common offset
    x, res, gamma, beta, kp, dsc = _ln_case(65, 768, 0.1, offset=True, const=True)
    f = R.ln_forward(x, gamma, beta, eps=1e-5, residual=res, kp=kp, dscale=dsc)
    b = R.ln_forward_bounds(f, R.U_BF16)
    rstd_bad = 1.0 / (torch.sqrt(f["var"][:, 0]) + 1e-5)
    assert R.exceeds(rstd_bad, f["rstd"], b["rstd"])


def _ln_bwd_case(rows, C, drop, seed=1):
    x, res, gamma, beta, kp, dsc = _ln_case(rows, C, drop, seed=seed)
    f = R.ln_forward(x, gamma, beta, eps=1e-5, residual=res, kp=kp, dscale=dsc)
    dy = torch.randn(rows, C, generator=_gen(seed + 10), dtype=F64)
    return f, dy, gamma, kp, dsc


def test_ln_dxsum_of_ds_under_dropout_leaves_bound():
    f, dy, gamma, kp, dsc = _ln_bwd_case(64, 768, 0.1)
    b = R.ln_backward(dy, f["s"], f["mean"], f["rstd"], gamma, kp=kp, dscale=dsc)
    bb = R.ln_backward_bounds(b, R.U_BF16)
    assert R.exceeds(b["ds"].sum(0), b["dxsum"], bb["dxsum"])


@pytest.mark.parametrize("rows", [16 * SMS + 1, 16 * SMS - 1, 10007])
def test_ln_dgamma_missing_last_row_of_a_warp_leaves_bound(rows):
    """The persistent backward: warp w of the grid (2 SMs CTAs x 8 warps) visits rows w, w + stride, ...; a dgamma that
    drops the last row each warp visits."""
    f, dy, gamma, kp, dsc = _ln_bwd_case(rows, 256, 0.0)
    b = R.ln_backward(dy, f["s"], f["mean"], f["rstd"], gamma)
    bb = R.ln_backward_bounds(b, R.U_BF16)
    stride = 16 * SMS
    last = torch.zeros(rows, dtype=torch.bool)
    for w in range(min(stride, rows)):
        last[w + (rows - 1 - w) // stride * stride] = True
    bad = (b["dy"] * b["xhat"])[~last].sum(0)
    assert R.exceeds(bad, b["dgamma"], bb["dgamma"])


def _bn_case(rows, C, training=True, act="tanh", seed=2):
    g = _gen(seed)
    x = torch.randn(rows, C, generator=g, dtype=F64) * 1.5 + 0.3
    gamma = 1.0 + 0.3 * torch.randn(C, generator=g, dtype=F64)
    beta = 0.3 * torch.randn(C, generator=g, dtype=F64)
    rm = torch.randn(C, generator=g, dtype=F64)
    rv = torch.rand(C, generator=g, dtype=F64) + 0.5
    f = R.bn_forward(x, gamma, beta, rm, rv, training=training, momentum=0.1, eps=1e-5, act_name=act)
    return x, gamma, beta, rm, rv, f


def test_bn_defects_leave_bounds():
    # biased running variance (rows = 256, fp32)
    x, gamma, beta, rm, rv, f = _bn_case(256, 80)
    b = R.bn_forward_bounds(f, R.U32)
    bad = 0.9 * rv + 0.1 * f["var"]
    assert R.exceeds(bad, f["running_var"], b["running_var"])
    # eval mode normalising with the batch statistics (bf16)
    x, gamma, beta, rm, rv, fe = _bn_case(255, 80, training=False)
    b = R.bn_forward_bounds(fe, R.U_BF16)
    ft = R.bn_forward(x, gamma, beta, rm, rv, training=True, momentum=0.1, eps=1e-5, act_name="tanh")
    assert R.exceeds(ft["y"], fe["y"], b["y"])
    # dx without its mean(g) term (32769 rows: past the row-block cap)
    x, gamma, beta, rm, rv, f = _bn_case(128 * 256 + 1, 37, act="none")
    dy = torch.randn(x.shape, generator=_gen(11), dtype=F64) + 0.2
    bw = R.bn_backward(dy, x, f["pre"], gamma, f["mean"], f["rstd"])
    bb = R.bn_backward_bounds(bw, R.U32)
    rows = x.shape[0]
    bad = bw["gamma"] * bw["rstd"] * (bw["g"] - bw["xhat"] * bw["sgx"] / rows)
    assert R.exceeds(bad, bw["dx"], bb["dx"])


def _pe_case(seed=3):
    B, T, C, V, pad = 3, 40, 64, 50, 1
    g = _gen(seed)
    tokens = torch.randint(0, V, (B, T), generator=g)
    tokens[0, :6] = 7
    tokens[2, -9:] = pad
    pe = torch.randn(B * T + 8, C, generator=g, dtype=F64)
    emb = torch.randn(V, C, generator=g, dtype=F64)
    return B, T, C, V, pad, tokens, pe, emb


def test_posenc_defects_leave_bounds():
    B, T, C, V, pad, tokens, pe, emb = _pe_case()
    y, bnd = R.posenc_forward(pe, 1.3, T, tokens=tokens, emb=emb, u=R.U_BF16)
    bad = emb.to(F64)[tokens] + 1.3 * pe[:B * T].view(B, T, C)  # pe indexed by b T + t
    assert R.exceeds(bad, y, bnd)
    dy = torch.randn(B, T, C, generator=_gen(12), dtype=F64)
    b = R.posenc_backward(dy, pe, T, tokens=tokens, padding_idx=pad, n_emb=V)
    bad = torch.zeros(V, C, dtype=F64).index_add_(0, tokens.reshape(-1), dy.reshape(-1, C))  # padding_idx included
    assert R.exceeds(bad, b["demb"], b["b_demb"])


def test_colsum_row_counted_into_next_group_leaves_bound():
    x = torch.randn(1000, 96, generator=_gen(6), dtype=F64)
    gr = 300
    ref, bnd = R.colsum(x, gr)
    bad = torch.stack([x[max(0, g * gr - 1):(g + 1) * gr - 1].sum(0) for g in range(4)])
    assert R.exceeds(bad, ref, bnd)


def test_relu_grad_at_zero_and_lrelu_phase_leave_bounds():
    x = torch.tensor([-1.0, 0.0, -0.0, 2.0], dtype=F64)
    g = torch.ones(4, dtype=F64)
    ref, bnd = R.act_bwd_bound(g, x, "relu", R.U_BF16)
    assert R.exceeds(torch.where(x >= 0, g, 0 * g), ref, bnd)
    xx = torch.randn(2, 14, 8, generator=_gen(8), dtype=F64)
    want = R.lrelu_pad(xx, 6, 2, 1, 2, 0.1)
    assert R.exceeds(R.lrelu_pad(xx, 6, 2, 0, 2, 0.1), want, R.U_BF16 * want.abs() + R.TINY)


def _adam_case(n=1027, step=3, wd=0.1, lr=0.05, gmul=0.5, max_norm=1.0, seed=9):
    g0 = _gen(seed)
    p = torch.randn(n, generator=g0).double()
    g = torch.randn(n, generator=g0).double()
    m = 0.1 * torch.randn(n, generator=g0).double()
    v = 0.01 * torch.rand(n, generator=g0).double()
    kw = dict(lr=lr, beta1=0.9, beta2=0.98, eps=1e-6, weight_decay=wd, step=step)
    gn2 = float(R.f32(float((g * g).sum())))
    out = R.adam_step(p, g, m, v, **kw, grad_norm_sq=gn2, max_norm=max_norm, grad_mul=gmul)
    bnd = R.adam_bounds((p, m, v), out, **kw, device_step=True)
    return p, g, m, v, kw, gn2, out, bnd


def test_adam_defects_leave_bounds():
    p, g, m, v, kw, gn2, out, bnd = _adam_case()
    lr, wd, ss = R.f32(kw["lr"]), R.f32(kw["weight_decay"]), out["step_size"]
    den = torch.sqrt(out["v"]) + R.f32(kw["eps"])
    # weight decay after the update
    bad = (p - ss * out["m"] / den) * (1 - wd * lr)
    assert R.exceeds(bad, out["p"], bnd["p"])
    # bias correction without the square root
    b1, b2, t = R.f32(0.9), R.f32(0.98), kw["step"]
    bad = p * (1 - wd * lr) - lr * (1 - b2 ** t) / (1 - b1 ** t) * out["m"] / den
    assert R.exceeds(bad, out["p"], bnd["p"])
    # clip norm without grad_mul (clip active at max_norm = 1: |g| ~ 32)
    bad_out = R.adam_step(p, g, m, v, **kw, grad_norm_sq=gn2 / 0.25, max_norm=1.0, grad_mul=0.5)
    assert R.exceeds(bad_out["m"], out["m"], bnd["m"])
    # an update applied on an inf norm: the kernel must leave p as it was
    assert R.exceeds(out["p"], p, R.TINY + 0 * p)
    # the last n % 4 elements skipped
    bad = out["p"].clone()
    bad[-3:] = p[-3:]
    assert R.exceeds(bad, out["p"], bnd["p"])

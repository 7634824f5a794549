"""-m gpu: the dropout mask of every drop site, read back from the kernel's output and compared bit for bit with
tests/dropout_ref.py (Philox4x32-7(seed, offset, i / 8), lane i % 8, threshold p * 65536), forward and backward.

Every site computes its index its own way -- (z * M + m) * N + n in the GEMM epilogue (test_gemm_contract_gpu.py),
the linear element index in st5_dropout / st5_act_bwd / posenc, row * C + c in the norms (whatever the row pitches),
((b * H + h) * Tq + i) * round_up(Tk, 32) + j for attention probabilities -- and a backward that disagrees with its
forward trains wrong without any error. The inputs are chosen so that the output IS the mask (x = 1, residual = 0;
uniform attention probabilities with V / dO one-hot blocks), or the backward is compared elementwise with fp64
formulas that apply the expected mask."""
import math

import numpy as np
import pytest
import torch

import dropout_ref as D

pytestmark = pytest.mark.gpu

SEED = 0x1_2345_6789  # more than 32 bits: the high word is key word k1
OFFSET = (5 << 32) + 3  # the high word goes to counter word c3


def _keep(n, p, seed=SEED, offset=OFFSET, shape=None):
    m = torch.from_numpy(D.keep_mask(seed, offset, np.arange(n, dtype=np.uint64), p))
    return m.reshape(shape) if shape is not None else m


def _check_mask(got, keep, p, dtype, what):
    got = got.detach().double().cpu()
    assert torch.equal(got != 0, keep), (f"{what}: {int(((got != 0) != keep).sum())} of {keep.numel()} keep decisions "
                                         f"differ from dropout_ref")
    scale = torch.tensor(D.drop_scale(p), dtype=torch.float32).to(dtype).double()
    assert bool((got[keep] == scale).all()), f"{what}: kept values are not 1 / (1 - p)"


@pytest.fixture(autouse=True)
def _bf16_runtime():
    from speecht5_b200.ops import RT
    saved = (RT.dtype, RT.attn_tensor_core, RT.attn_fused, RT.attn_fused_bwd, RT.attn_flash, RT.ffn_gate,
             RT.fp32_stream, RT._seed_t, RT._seed, RT._offset)
    RT.disable_device_seed()
    yield RT
    (RT.dtype, RT.attn_tensor_core, RT.attn_fused, RT.attn_fused_bwd, RT.attn_flash, RT.ffn_gate,
     RT.fp32_stream, RT._seed_t, RT._seed, RT._offset) = saved
    RT.invalidate_shadows()


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])


# ------------------------------------------------------------------------------------------------ elementwise kernels
@DTYPES
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_and_act_bwd(cuda, dtype, p):
    """st5_dropout(ones) is the mask; st5_act_bwd(dy = ones, pre) = mask * scale * act'(pre), same index."""
    from speecht5_b200 import kernels as K
    n = 100_003
    x = torch.ones(n, device=cuda, dtype=dtype)
    y = torch.empty_like(x)
    K.dropout(x, y, p, SEED, OFFSET)
    keep = _keep(n, p)
    _check_mask(y, keep, p, dtype, "st5_dropout")
    pre = torch.full((n,), 2.0, device=cuda, dtype=dtype)  # relu'(2) = 1
    d = torch.empty_like(x)
    K.act_bwd(x, pre, d, "relu", drop_p=p, seed=SEED, offset=OFFSET)
    _check_mask(d, keep, p, dtype, "st5_act_bwd")


# ------------------------------------------------------------------------------------------------ LayerNorm
@DTYPES
@pytest.mark.parametrize("C", [256, 768, 1024])
@pytest.mark.parametrize("rows", [40, 100])  # st5_ln_bwd: two kernels below 64 rows, one fused kernel from 64
@pytest.mark.parametrize("stream", [False, True], ids=["plain", "fp32_stream"])
def test_layer_norm_forward_and_backward_masks(cuda, dtype, C, rows, stream):
    """s = residual + dropout(x) with x = 1, residual = 0 is the mask (index row * C + c); the backward's
    dx = ds * mask / (1 - p) at the same index."""
    from speecht5_b200 import kernels as K
    p = 0.1
    x = torch.ones(rows, C, device=cuda, dtype=dtype)
    res = torch.zeros_like(x)
    gamma = torch.ones(C, device=cuda)
    beta = torch.zeros(C, device=cuda)
    y, s = torch.empty_like(x), torch.empty_like(x)
    mean, rstd = torch.empty(rows, device=cuda), torch.empty(rows, device=cuda)
    kw = dict(residual_f32=torch.zeros(rows, C, device=cuda), y_f32=torch.empty(rows, C, device=cuda)) if stream else {}
    K.ln_fwd(x, None if stream else res, gamma, beta, y, s, mean, rstd, 1e-5, p, SEED, OFFSET, **kw)
    keep = _keep(rows * C, p, shape=(rows, C))
    _check_mask(s, keep, p, dtype, "ln_fwd" + ("_stream" if stream else ""))
    # backward on a non-degenerate s
    torch.manual_seed(rows + C)
    s2 = (torch.randn(rows, C, device=cuda) + 0.5).to(dtype)
    mean2 = s2.float().mean(-1)
    rstd2 = 1.0 / torch.sqrt(s2.float().var(-1, unbiased=False) + 1e-5)
    dy = torch.randn(rows, C, device=cuda).to(dtype)
    ds, dx = torch.empty_like(dy), torch.empty_like(dy)
    dg, db = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
    K.ln_bwd(dy, s2, mean2, rstd2, gamma, ds, dx, dg, db, p, SEED, OFFSET)
    dsd, dxd = ds.double().cpu(), dx.double().cpu()
    want = torch.where(keep, dsd * D.drop_scale(p), torch.zeros_like(dsd))
    tol = 1e-6 if dtype == torch.float32 else 2.0 ** -7
    assert bool(((dxd - want).abs() <= tol * want.abs() + 1e-30).all()), "ln_bwd: dx != ds * mask / (1 - p)"
    sure = dsd.abs() > 1e-20
    assert torch.equal((dxd != 0)[sure], keep[sure])


# ------------------------------------------------------------------------------------------------ posenc
@DTYPES
@pytest.mark.parametrize("C", [64, 37])  # 8-channel vector kernel / scalar kernel
def test_posenc_forward_and_backward_masks(cuda, dtype, C):
    from speecht5_b200 import kernels as K
    p, B, T = 0.2, 3, 41
    x = torch.ones(B, T, C, device=cuda, dtype=dtype)
    pe = torch.zeros(T, C, device=cuda)
    alpha = torch.zeros(1, device=cuda)
    y = torch.empty_like(x)
    K.posenc_fwd(None, None, x, pe, alpha, y, p, SEED, OFFSET)
    keep = _keep(B * T * C, p, shape=(B, T, C))
    _check_mask(y, keep, p, dtype, "posenc_fwd")
    dx = torch.empty_like(x)
    dalpha = torch.zeros(1, device=cuda)
    K.posenc_bwd(x, None, -1, pe, dx, None, dalpha, p, SEED, OFFSET)
    _check_mask(dx, keep, p, dtype, "posenc_bwd")


# ------------------------------------------------------------------------------------------------ BatchNorm
@pytest.mark.parametrize("C", [80, 37])  # vector kernels / scalar kernels
def test_batch_norm_forward_and_backward_masks(cuda, C):
    """y = dropout(BN(x)) with gamma = 0, beta = 1 is the mask. The index is the LOGICAL row * C + c, whatever the row
    pitches x_ld / y_ld / dy_ld / dx_ld are (here all different from C). The backward is checked elementwise against
    the fp64 BatchNorm backward of g = dy * mask / (1 - p)."""
    from speecht5_b200 import kernels as K
    p, rows = 0.3, 150
    ld = C + 8 if C % 8 == 0 else C + 3
    dev = cuda
    x = torch.randn(rows, ld, device=dev)
    gamma0, beta1 = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    sm, sr = torch.empty(C, device=dev), torch.empty(C, device=dev)
    y = torch.zeros(rows, ld + 8, device=dev)
    scratch = torch.empty(2 * C, device=dev)
    K.bn_fwd(x, ld, gamma0, beta1, rm, rv, sm, sr, y, ld + 8, None, rows, C, True, 0.1, 1e-5, None, p, SEED, OFFSET,
             scratch)
    keep = _keep(rows * C, p, shape=(rows, C))
    _check_mask(y[:, :C], keep, p, torch.float32, "bn_fwd")
    assert bool((y[:, C:] == 0).all())
    # backward
    torch.manual_seed(C)
    gamma = torch.rand(C, device=dev) + 0.5
    dy = torch.randn(rows, ld + 16, device=dev)
    dx = torch.full((rows, ld + 8), float("nan"), device=dev)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    K.bn_bwd(dy, ld + 16, x, ld, None, gamma, sm, sr, dx, ld + 8, dg, db, rows, C, None, p, SEED, OFFSET, scratch)
    xs = x[:, :C].double().cpu()
    mu, rs = sm.double().cpu(), sr.double().cpu()
    xh = (xs - mu) * rs
    g = torch.where(keep, dy[:, :C].double().cpu() * D.drop_scale(p), torch.zeros(rows, C, dtype=torch.float64))
    want = gamma.double().cpu() * rs * (g - g.mean(0) - xh * (g * xh).mean(0))
    got = dx[:, :C].double().cpu()
    assert bool(((got - want).abs() <= 1e-4 * (g.abs().mean(0) + want.abs()) * gamma.double().cpu() * rs).all())
    assert torch.allclose(db.double().cpu(), g.sum(0), rtol=1e-5, atol=1e-4)


# ------------------------------------------------------------------------------------------------ attention
IMPLS = ["rows", "tc", "fused", "flash"]


def _route(RT, impl):
    RT.dtype = torch.bfloat16
    RT.attn_tensor_core = impl != "rows"
    RT.attn_fused = RT.attn_fused_bwd = impl in ("fused", "flash")
    RT.attn_flash = "all" if impl == "flash" else False


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("Tk", [29, 64, 160, 313, 499])
@pytest.mark.parametrize("mask", ["key_pad", "causal"])
def test_attention_masks_forward_and_backward(cuda, _bf16_runtime, impl, Tk, mask):
    """q = 0: the probabilities are uniform over the unmasked keys. V one-hot on key block kb (V[j, c] = [j == 64 kb + c]
    in every head) makes out[i, c] the dropped probability of key 64 kb + c; dO one-hot on query block qb makes
    dV[j, c] = sum_i P_drop[i, j] dO[i, c] the dropped probability of query 64 qb + c -- so the backward's own mask (the
    row kernels' and attention_tc.cu's regenerated one, the sign bits of psave in the fused backward) is read too."""
    from speecht5_b200 import ops
    RT = _bf16_runtime
    if impl == "fused" and Tk > 320:
        pytest.skip("the resident fused kernel holds Tk <= 320 (longer rows stream through attention_flash.cu)")
    _route(RT, impl)
    p, B, H = 0.2, 2, 2
    d = 64 * H
    Tq = Tk if mask == "causal" else 70
    dev = cuda
    lens = torch.tensor([Tk, Tk - 7])
    key_pad = (torch.arange(Tk)[None, :] >= lens[:, None]).to(dev) if mask == "key_pad" else None
    i = torch.arange(Tq)[:, None]
    j = torch.arange(Tk)[None, :]
    valid = torch.ones(B, 1, Tq, Tk, dtype=torch.bool)
    if mask == "causal":
        valid &= (j <= i)[None, None]
    else:
        valid &= (j[None] < lens[:, None, None])[:, None]
    n_valid = valid.sum(-1, keepdim=True).double()
    nkb, nqb = (Tk + 63) // 64, (Tq + 63) // 64
    torch.manual_seed(Tk)
    kbase = torch.randn(B, Tk, d)
    for run in range(max(nkb, nqb)):
        kb, qb = run % nkb, run % nqb
        q_buf = torch.zeros(B, Tq, d, device=dev, dtype=torch.bfloat16, requires_grad=True)
        v = torch.zeros(B, Tk, H, 64)
        jj = torch.arange(64 * kb, min(64 * kb + 64, Tk))
        v[:, jj, :, jj - 64 * kb] = 1.0
        kv = torch.cat([kbase, v.reshape(B, Tk, d)], -1).to(dev, torch.bfloat16).requires_grad_()
        RT.manual_seed(11)
        off0 = RT._offset
        out, _ = ops.attention(q_buf, kv, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=key_pad,
                               causal=mask == "causal", drop_p=p)
        assert RT._offset == off0 + 1
        keep = torch.from_numpy(D.attn_keep(RT.seed, off0 + 1, p, B, H, Tq, Tk)) & valid
        P = torch.where(keep, D.drop_scale(p) / n_valid, torch.zeros(()).double())  # [B, H, Tq, Tk]
        got = out.detach().double().cpu().reshape(B, Tq, H, 64)[..., :len(jj)].permute(0, 2, 1, 3)  # [B, H, Tq, c]
        want = P[..., jj]
        where = f"{impl} Tk={Tk} {mask} forward, keys {int(jj[0])}..{int(jj[-1])}"
        assert torch.equal(got != 0, want != 0), f"{where}: {int(((got != 0) != (want != 0)).sum())} decisions differ"
        assert bool(((got - want).abs() <= 2.0 ** -7 * want).all()), where
        dO = torch.zeros(B, Tq, H, 64)
        ii = torch.arange(64 * qb, min(64 * qb + 64, Tq))
        dO[:, ii, :, ii - 64 * qb] = 1.0
        out.backward(dO.reshape(B, Tq, d).to(dev, torch.bfloat16))
        dv = kv.grad.double().cpu()[..., d:].reshape(B, Tk, H, 64)[..., :len(ii)].permute(0, 2, 3, 1)  # [B, H, c, Tk]
        want = P[:, :, ii, :]
        where = f"{impl} Tk={Tk} {mask} backward (dV), queries {int(ii[0])}..{int(ii[-1])}"
        assert torch.equal(dv != 0, want != 0), f"{where}: {int(((dv != 0) != (want != 0)).sum())} decisions differ"
        assert bool(((dv - want).abs() <= 2.0 ** -6 * want).all()), where


# ------------------------------------------------------------------------------------------------ module level
@DTYPES
@pytest.mark.parametrize("act", ["gelu", None])
def test_linear_dropout_forward_and_backward(cuda, _bf16_runtime, dtype, act):
    """ops.linear with drop_p, N = 330 so that the output pitch (336) differs from N: the forward mask is the GEMM
    epilogue's (index m * N + n), the backward regenerates it in st5_act_bwd / st5_dropout on the compacted gradient.
    Compared elementwise with fp64 autograd of the same operands applying the expected mask."""
    from speecht5_b200 import ops
    RT = _bf16_runtime
    RT.dtype = dtype
    RT.invalidate_shadows()
    p, M, Kd, N = 0.3, 150, 96, 330
    torch.manual_seed(3)
    W = torch.nn.Parameter(torch.randn(N, Kd, device=cuda) * Kd ** -0.5)
    b = torch.nn.Parameter(torch.randn(N, device=cuda) * 0.1)
    x = torch.randn(M, Kd, device=cuda).to(dtype).requires_grad_()
    RT.manual_seed(21)
    off0 = RT._offset
    y = ops.linear(x, (W,), (b,), act=act, drop_p=p)
    assert RT._offset == off0 + 1
    g = torch.randn(M, N, device=cuda).to(dtype)
    y.backward(g)
    keep = _keep(M * N, p, seed=RT.seed, offset=off0 + 1, shape=(M, N))
    wd = W.detach().double().cpu() if dtype == torch.float32 else W.detach().to(torch.bfloat16).double().cpu()
    xr = x.detach().double().cpu().requires_grad_()
    Wr = wd.clone().requires_grad_()
    pre = xr @ Wr.t() + b.detach().double().cpu()
    from gemm_emulator import _act
    a = _act(pre, None if act is None else ("gelu" if dtype == torch.float32 else "gelu_tanh"))
    yr = torch.where(keep, a * D.drop_scale(p), torch.zeros_like(a))
    yr.backward(g.double().cpu())
    mag = xr.detach().abs() @ wd.abs().t()
    if dtype == torch.float32:  # three-pass bf16 split: products good to ~2^-16
        ybound = 2.0 ** -14 * (mag + 1) * 2
    else:
        ybound = 2.0 ** -8 * yr.detach().abs() + 2.0 ** -9 * (mag + 1) * 2
    err = (y.detach().double().cpu() - yr.detach()).abs()
    assert bool((err <= ybound).all()), f"forward: {int((err > ybound).sum())} elements off"
    sure = a.detach().abs() > 1e-2  # (the kept set itself, where the undropped value is clearly non-zero)
    assert torch.equal((y.detach().cpu() != 0)[sure], keep[sure]), "forward: kept set differs from dropout_ref"
    gm = g.double().cpu().abs() * keep * D.drop_scale(p) * 1.2
    dxb = (2.0 ** -13 if dtype == torch.float32 else 2.0 ** -6) * (gm @ wd.abs()) + 1e-12
    e = (x.grad.double().cpu() - xr.grad).abs()
    assert bool((e <= dxb).all()), f"dx: {int((e > dxb).sum())} elements off"
    dwb = (2.0 ** -13 if dtype == torch.float32 else 2.0 ** -6) * (gm.t() @ xr.detach().abs()) + 1e-12
    e = (W.grad.double().cpu() - Wr.grad).abs()
    assert bool((e <= dwb).all()), f"dW: {int((e > dwb).sum())} elements off"


def _within(got, ref, bound, what):
    got = got.detach().double().cpu()
    bad = ~((got - ref).abs() <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at "
                                 f"{tuple(int(i) for i in bad.nonzero()[0])}")


def _row_bound(ref, tol):
    """Elementwise bound with a floor of the mean magnitude of the element's row (last dimension)."""
    a = ref.abs()
    return tol * (a + a.mean(-1, keepdim=True)) + 1e-30


MODES = pytest.mark.parametrize("mode", ["f32", "bf16"])


@pytest.mark.parametrize("mode", ["f32", "bf16_gate", "bf16_nogate"])
def test_ffn_dropout_forward_and_backward(cuda, _bf16_runtime, mode):
    """FFNFn with drop_a and drop_o: fc1's epilogue draws mask a at index m * F + f (offset n + 1), fc2's mask o at
    m * D + d (offset n + 2). Backward: st5_dropout regenerates mask o; the dH GEMM regenerates mask a in its epilogue
    (non-gate path) or multiplies by the gate fc1 stored, keep * scale * gelu_tanh'(pre) (RT.ffn_gate, bf16). Forward
    masks are read from the saved activations; everything is compared elementwise with fp64 formulas applying them."""
    from gemm_emulator import _act, _act_grad
    from speecht5_b200 import ops
    RT = _bf16_runtime
    dtype = torch.float32 if mode == "f32" else torch.bfloat16
    RT.dtype = dtype
    RT.ffn_gate = mode == "bf16_gate"
    RT.invalidate_shadows()
    pa, po, B, T, Dm, F = 0.2, 0.1, 3, 50, 128, 256
    M = B * T
    torch.manual_seed(5)
    fc1, fc2 = torch.nn.Linear(Dm, F).to(cuda), torch.nn.Linear(F, Dm).to(cuda)
    x = torch.randn(B, T, Dm, device=cuda).to(dtype).requires_grad_()
    RT.manual_seed(31)
    off0 = RT._offset
    o = ops.ffn(x, fc1, fc2, "gelu", drop_a=pa, drop_o=po)
    assert RT._offset == off0 + 2
    _, h_saved, pre_saved = (t.detach().double().cpu() for t in o.grad_fn.saved_tensors)
    g = torch.randn(B, T, Dm, device=cuda).to(dtype)
    o.backward(g)
    ka = _keep(M * F, pa, seed=RT.seed, offset=off0 + 1, shape=(M, F))
    ko = _keep(M * Dm, po, seed=RT.seed, offset=off0 + 2, shape=(M, Dm))
    cast = (lambda t: t.detach().double().cpu()) if dtype == torch.float32 else \
        (lambda t: t.detach().to(torch.bfloat16).double().cpu())
    W1, W2 = cast(fc1.weight), cast(fc2.weight)
    b1, b2 = fc1.bias.detach().double().cpu(), fc2.bias.detach().double().cpu()
    xs = x.detach().double().cpu().reshape(M, Dm)
    act = "gelu" if dtype == torch.float32 else "gelu_tanh"
    sa, so = D.drop_scale(pa), D.drop_scale(po)
    pre = xs @ W1.t() + b1
    h = torch.where(ka, _act(pre, act) * sa, torch.zeros(()).double())
    q = h @ W2.t() + b2
    o_ref = torch.where(ko, q * so, torch.zeros(()).double())
    gd = g.double().cpu().reshape(M, Dm)
    go = torch.where(ko, gd * so, torch.zeros(()).double())
    dpre = torch.where(ka, (go @ W2) * sa, torch.zeros(()).double()) * _act_grad(pre, act)
    # forward masks, read from what the kernels stored
    sure = _act(pre, act).abs() > 1e-2
    assert torch.equal((h_saved != 0)[sure], ka[sure]), "fc1 epilogue: mask a differs from dropout_ref"
    if mode == "bf16_gate":  # the stored gate keep * scale * gelu_tanh'(pre)
        sure = _act_grad(pre, act).abs() > 1e-2
        assert torch.equal((pre_saved != 0)[sure], ka[sure]), "fc1 gate: mask a differs from dropout_ref"
    sure = q.abs() > 1e-2
    assert torch.equal((o.detach().cpu().reshape(M, Dm) != 0)[sure], ko[sure]), "fc2 epilogue: mask o differs"
    # elementwise bounds from the magnitudes of the terms
    tol = 2.0 ** -12 if dtype == torch.float32 else 2.0 ** -5
    rnd = 0.0 if dtype == torch.float32 else 2.0 ** -7
    hm = h.abs() + sa * 1.2 * (xs.abs() @ W1.abs().t() + b1.abs())
    _within(o.reshape(M, Dm), o_ref, tol * so * (hm @ W2.abs().t() + b2.abs()) + rnd * o_ref.abs(), "o")
    dpm = sa * 1.2 * (go.abs() @ W2.abs())
    dx_ref = dpre @ W1
    _within(x.grad.reshape(M, Dm), dx_ref, tol * (dpm @ W1.abs()) + rnd * dx_ref.abs() + 1e-30, "dx")
    _within(fc1.weight.grad, dpre.t() @ xs, tol * (dpm.t() @ xs.abs()) + 1e-30, "dW1")
    _within(fc1.bias.grad, dpre.sum(0), tol * dpm.sum(0) + 1e-30, "db1")
    _within(fc2.weight.grad, go.t() @ h, tol * (go.abs().t() @ hm) + 1e-30, "dW2")
    _within(fc2.bias.grad, go.sum(0), tol * go.abs().sum(0) + 1e-30, "db2")


@pytest.mark.parametrize("mode", ["f32", "bf16", "bf16_stream"])
def test_residual_layer_norm_dropout(cuda, _bf16_runtime, mode):
    """y = LayerNorm(residual + dropout(x)) forward and backward against fp64 autograd with the expected mask (index
    row * C + c); bf16_stream adds the fp32 residual stream (fp32 residual in, fp32 copy of y out)."""
    from speecht5_b200 import ops
    RT = _bf16_runtime
    dtype = torch.float32 if mode == "f32" else torch.bfloat16
    RT.dtype = dtype
    RT.fp32_stream = mode == "bf16_stream"
    p, B, T, C = 0.2, 3, 30, 256
    torch.manual_seed(7)
    ln = torch.nn.LayerNorm(C).to(cuda)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5)
        ln.bias.uniform_(-0.5, 0.5)
    xv = torch.randn(B, T, C, device=cuda)
    x = (xv.sign() * (0.5 + xv.abs())).to(dtype).requires_grad_()  # |x| >= 0.5: a wrong keep bit moves s by >= 0.5
    r32 = torch.randn(B, T, C, device=cuda)
    r = r32.to(dtype).requires_grad_()
    if mode == "bf16_stream":
        r._st5_f32 = r32.contiguous()
    RT.manual_seed(3)
    off0 = RT._offset
    y = ops.residual_layer_norm(x, r, ln, drop_p=p, stream=mode == "bf16_stream")
    assert RT._offset == off0 + 1
    g = torch.randn(B, T, C, device=cuda).to(dtype)
    y.backward(g)
    keep = _keep(B * T * C, p, seed=RT.seed, offset=off0 + 1, shape=(B, T, C))
    xr = x.detach().double().cpu().requires_grad_()
    rr = (r32 if mode == "bf16_stream" else r.detach()).double().cpu().requires_grad_()
    w = ln.weight.detach().double().cpu().requires_grad_()
    bb = ln.bias.detach().double().cpu().requires_grad_()
    s = rr + torch.where(keep, xr * D.drop_scale(p), torch.zeros(()).double())
    yr = torch.nn.functional.layer_norm(s, (C,), w, bb, ln.eps)
    yr.backward(g.double().cpu())
    tol = 1e-5 if dtype == torch.float32 else 2.0 ** -6
    _within(y, yr.detach(), _row_bound(yr.detach(), tol), "y")
    if mode == "bf16_stream":
        _within(y._st5_f32, yr.detach(), _row_bound(yr.detach(), 1e-5), "y_f32")
    gt = 1e-4 if dtype == torch.float32 else 2.0 ** -5
    _within(x.grad, xr.grad, _row_bound(xr.grad, gt), "dx")
    _within(r.grad, rr.grad, _row_bound(rr.grad, gt), "dresidual")
    _within(ln.weight.grad, w.grad, gt * w.grad.abs() + gt * w.grad.abs().mean(), "dgamma")
    _within(ln.bias.grad, bb.grad, gt * bb.grad.abs() + gt * bb.grad.abs().mean(), "dbeta")


@MODES
def test_scaled_posenc_dropout(cuda, _bf16_runtime, mode):
    """y = dropout(x + alpha * pe[:T]) (index (b * T + t) * C + c) and its backward (dx, dalpha)."""
    from speecht5_b200 import ops
    RT = _bf16_runtime
    dtype = torch.float32 if mode == "f32" else torch.bfloat16
    RT.dtype = dtype
    p, B, T, C = 0.3, 2, 37, 64
    torch.manual_seed(8)
    pe = torch.randn(T + 5, C, device=cuda)
    alpha = torch.nn.Parameter(torch.tensor(1.3, device=cuda))
    x = torch.randn(B, T, C, device=cuda).to(dtype).requires_grad_()
    RT.manual_seed(4)
    off0 = RT._offset
    y = ops.scaled_posenc(pe, alpha, p, x=x)
    assert RT._offset == off0 + 1
    g = torch.randn(B, T, C, device=cuda).to(dtype)
    y.backward(g)
    keep = _keep(B * T * C, p, seed=RT.seed, offset=off0 + 1, shape=(B, T, C))
    sc = D.drop_scale(p)
    pe_d = pe[:T].double().cpu()
    v = x.detach().double().cpu() + 1.3 * pe_d
    y_ref = torch.where(keep, v * sc, torch.zeros(()).double())
    tol = 1e-6 if dtype == torch.float32 else 2.0 ** -7
    _within(y, y_ref, tol * sc * (x.detach().double().cpu().abs() + 1.3 * pe_d.abs()) + 1e-30, "y")
    gk = torch.where(keep, g.double().cpu() * sc, torch.zeros(()).double())
    _within(x.grad, gk, tol * gk.abs() + 1e-30, "dx")
    _within(alpha.grad, (gk * pe_d).sum(), 1e-4 * (gk * pe_d).abs().sum(), "dalpha")


@MODES
def test_batch_norm_act_dropout(cuda, _bf16_runtime, mode):
    """dropout(tanh(BatchNorm1d(x))) in training mode, forward and backward against fp64 autograd with the expected
    mask at index row * C + c."""
    from speecht5_b200 import ops
    RT = _bf16_runtime
    dtype = torch.float32 if mode == "f32" else torch.bfloat16
    RT.dtype = dtype
    p, B, T, C = 0.5, 3, 40, 80
    torch.manual_seed(9)
    bn = torch.nn.BatchNorm1d(C).to(cuda)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.3, 0.3)
    x = (torch.randn(B, T, C, device=cuda) * 2 + 0.5).to(dtype).requires_grad_()
    RT.manual_seed(6)
    off0 = RT._offset
    y = ops.batch_norm_act(x, bn, True, act="tanh", drop_p=p)
    assert RT._offset == off0 + 1
    g = torch.randn(B, T, C, device=cuda).to(dtype)
    y.backward(g)
    keep = _keep(B * T * C, p, seed=RT.seed, offset=off0 + 1, shape=(B * T, C))
    xr = x.detach().double().cpu().reshape(B * T, C).requires_grad_()
    w = bn.weight.detach().double().cpu().requires_grad_()
    bb = bn.bias.detach().double().cpu().requires_grad_()
    z = torch.nn.functional.batch_norm(xr, None, None, w, bb, True, 0.0, bn.eps)
    yr = torch.where(keep, torch.tanh(z) * D.drop_scale(p), torch.zeros(()).double())
    yr.backward(g.double().cpu().reshape(B * T, C))
    tol = 1e-5 if dtype == torch.float32 else 2.0 ** -6
    _within(y.reshape(B * T, C), yr.detach(), tol * (yr.detach().abs() + 1), "y")
    gt = 1e-4 if dtype == torch.float32 else 2.0 ** -5
    dxa = xr.grad.abs()
    _within(x.grad.reshape(B * T, C), xr.grad, gt * (dxa + dxa.mean(0)), "dx")
    _within(bn.weight.grad, w.grad, gt * (w.grad.abs() + w.grad.abs().mean()), "dgamma")
    _within(bn.bias.grad, bb.grad, gt * (bb.grad.abs() + bb.grad.abs().mean()), "dbeta")


@MODES
@pytest.mark.parametrize("case", ["self_rpe", "self_causal", "cross_probs"])
def test_attention_dropout_module(cuda, _bf16_runtime, mode, case):
    """ops.attention with drop_p (RT's default routes: fused tensor-core kernels in bf16, row kernels in fp32) against
    fp64 autograd of softmax(scale q (k + pe)^T + masks) with the expected mask on P; returned probabilities undropped."""
    from speecht5_b200 import ops
    RT = _bf16_runtime
    dtype = torch.float32 if mode == "f32" else torch.bfloat16
    RT.dtype = dtype
    p, B, H, maxpos, scale = 0.2, 2, 2, 48, 0.125
    d = 64 * H
    Tq = 40
    Tk = 45 if case == "cross_probs" else Tq
    torch.manual_seed(10)
    pe = torch.nn.Parameter(torch.randn(2 * maxpos, 64, device=cuda) * 0.3) if case == "self_rpe" else None
    if case == "cross_probs":
        qb = (torch.randn(B, Tq, d, device=cuda) * 0.7).to(dtype).requires_grad_()
        kvb = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.7).to(dtype).requires_grad_()
        lens = torch.tensor([Tk, Tk - 9])
        key_pad = (torch.arange(Tk)[None, :] >= lens[:, None]).to(cuda)
        kw = dict(q_col=0, k_col=0, v_col=1, key_pad=key_pad, return_probs=True)
    else:
        qb = (torch.randn(B, Tq, 3 * d, device=cuda) * 0.7).to(dtype).requires_grad_()
        kvb, key_pad = None, None
        kw = dict(q_col=0, k_col=1, v_col=2, causal=case == "self_causal",
                  pe_k=pe, maxpos=maxpos if pe is not None else 0)
    RT.manual_seed(12)
    off0 = RT._offset
    out, probs = ops.attention(qb, kvb, H=H, d=d, scale=scale, drop_p=p, **kw)
    assert RT._offset == off0 + 1
    gout = torch.randn(B, Tq, d, device=cuda).to(dtype)
    loss = (out.float() * gout.float()).sum()
    gp = None
    if probs is not None:
        gp = torch.randn(probs.shape, device=cuda) * 0.1
        loss = loss + (probs.float() * gp).sum()
    loss.backward()
    keep = torch.from_numpy(D.attn_keep(RT.seed, off0 + 1, p, B, H, Tq, Tk))
    qr = qb.detach().double().cpu().requires_grad_()
    kvr = kvb.detach().double().cpu().requires_grad_() if kvb is not None else None
    per = pe.detach().double().cpu().requires_grad_() if pe is not None else None
    src = qr if kvr is None else kvr

    def heads(buf, col, T):
        return buf[..., col * d:(col + 1) * d].reshape(B, T, H, 64).transpose(1, 2)
    q = heads(qr, kw["q_col"], Tq) * scale
    k, v = heads(src, kw["k_col"], Tk), heads(src, kw["v_col"], Tk)
    s = q @ k.transpose(-1, -2)
    if per is not None:
        i, j = torch.arange(Tq)[:, None], torch.arange(Tk)[None, :]
        s = s + torch.einsum("bhic,ijc->bhij", q, per[(i - j).clamp(-maxpos, maxpos - 1) + maxpos])
    if case == "self_causal":
        s = s + torch.triu(torch.full((Tq, Tk), float("-inf"), dtype=torch.float64), 1)
    if key_pad is not None:
        s = s.masked_fill(key_pad.cpu()[:, None, None, :], float("-inf"))
    P = torch.softmax(s, -1)
    Pd = torch.where(keep, P * D.drop_scale(p), torch.zeros(()).double())
    o_ref = (Pd @ v).transpose(1, 2).reshape(B, Tq, d)
    loss_r = (o_ref * gout.double().cpu()).sum()
    if gp is not None:
        loss_r = loss_r + (P * gp.double().cpu()).sum()
    loss_r.backward()
    tol = 1e-4 if dtype == torch.float32 else 2.0 ** -5
    om = ((Pd.abs() @ v.abs()).transpose(1, 2).reshape(B, Tq, d)).detach()
    _within(out, o_ref.detach(), tol * om + 1e-30, "out")
    if probs is not None:
        _within(probs, P.detach(), tol * P.detach() + 1e-7, "probs")
    gt = 2e-4 if dtype == torch.float32 else 2.0 ** -4
    _within(qb.grad, qr.grad, _row_bound(qr.grad, gt), "dq_buf")
    if kvr is not None:
        _within(kvb.grad, kvr.grad, _row_bound(kvr.grad, gt), "dkv_buf")
    if per is not None:
        _within(pe.grad, per.grad, _row_bound(per.grad, gt), "dpe")

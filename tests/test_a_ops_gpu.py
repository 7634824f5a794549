"""-m gpu: every CUDA op (called through the C ABI) against a plain PyTorch fp32/fp64 statement of the same math."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.fixture(autouse=True)
def _mode():
    from speecht5_b200.ops import RT
    RT.dtype = torch.float32
    RT.manual_seed(1)
    RT.invalidate_shadows()
    yield
    RT.dtype = torch.bfloat16


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(4, 37, 768), (3, 5, 80), (2, 9, 1024), (7, 313, 768), (5, 67, 1024)])  # rows >= 64: fused dx + parameter pass
def test_layer_norm_residual(cuda, dtype, shape):
    from speecht5_b200 import ops
    ops.RT.dtype = dtype
    torch.manual_seed(0)
    C = shape[-1]
    ln = torch.nn.LayerNorm(C).to(cuda)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5); ln.bias.uniform_(-0.5, 0.5)
    x = torch.randn(shape, device=cuda).to(dtype).requires_grad_()
    r = torch.randn(shape, device=cuda).to(dtype).requires_grad_()
    y = ops.residual_layer_norm(x, r, ln)
    g = torch.randn(shape, device=cuda).to(dtype)
    y.backward(g)
    xr, rr = x.detach().double().requires_grad_(), r.detach().double().requires_grad_()
    lnr = torch.nn.LayerNorm(C).to(cuda).double()
    lnr.load_state_dict(ln.state_dict())
    yr = lnr(xr + rr)
    yr.backward(g.double())
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert rel(y, yr) < tol
    assert rel(x.grad, xr.grad) < tol and rel(r.grad, rr.grad) < tol
    assert rel(ln.weight.grad, lnr.weight.grad) < tol and rel(ln.bias.grad, lnr.bias.grad) < tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("rows,C,drop_p", [(10016, 768, 0.1), (5120, 768, 0.0), (333, 1024, 0.1), (40, 256, 0.0)])
def test_layer_norm_backward_column_sums_of_dx(cuda, dtype, rows, C, drop_p):
    """st5_ln_bwd's dxsum output (the producing projection's bias gradient, include/speecht5_b200.h): += column sums of
    the dx it writes, dropout included, for 16-byte aligned and unaligned targets; ds / dgamma / dbeta unchanged."""
    from speecht5_b200 import kernels as K
    torch.manual_seed(1)
    dy = torch.randn(rows, C, device=cuda).to(dtype)
    s = (torch.randn(rows, C, device=cuda) * 2 + 0.3).to(dtype)
    mean = s.float().mean(-1)
    rstd = 1.0 / torch.sqrt(s.float().var(-1, unbiased=False) + 1e-5)
    gamma = torch.rand(C, device=cuda) + 0.5
    for misalign in (0, 1):
        ds, dx = torch.empty_like(dy), (torch.empty_like(dy) if drop_p > 0 else None)
        dg, db = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
        buf = torch.full((C + 8,), 0.25, device=cuda)
        dxsum = buf[misalign:misalign + C]
        K.ln_bwd(dy, s, mean, rstd, gamma, ds, dx, dg, db, drop_p, 11, 5, dxsum=dxsum)
        ds2, dx2 = torch.empty_like(dy), (torch.empty_like(dy) if drop_p > 0 else None)
        dg2, db2 = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
        K.ln_bwd(dy, s, mean, rstd, gamma, ds2, dx2, dg2, db2, drop_p, 11, 5)
        if rows >= 64:  # (both calls take the fused kernel; below 64 rows the call without dxsum takes the two-kernel form)
            assert torch.equal(ds, ds2) and (dx is None or torch.equal(dx, dx2))
        else:
            assert rel(ds, ds2) < 1e-2 and (dx is None or rel(dx, dx2) < 1e-2)
        out = dx if dx is not None else ds
        want = out.double().sum(0) + 0.25
        # the kernel sums the un-rounded fp32 values, the check the rounded ones: allow the bf16 rounding of `rows` terms
        tol = 1e-4 if dtype == torch.float32 else 4e-3
        assert (dxsum.double() - want).abs().max() < tol * out.double().abs().sum(0).max(), (misalign,)
        assert rel(dg, dg2) < 1e-5 and rel(db, db2) < 1e-5
        xh = (s.float() - mean[:, None]) * rstd[:, None]
        assert rel(dg, (dy.float() * xh).sum(0)) < 1e-4 and rel(db, dy.float().sum(0)) < 1e-4
        assert float(buf[C + misalign:].sub(0.25).abs().max()) == 0 and float(buf[:misalign].sub(0.25).abs().sum()) == 0


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_linear_autograd(cuda, dtype):
    from speecht5_b200 import ops
    ops.RT.dtype = dtype
    torch.manual_seed(0)
    M, K, N = 200, 768, 328
    w1 = torch.nn.Parameter(torch.randn(N - 72, K, device=cuda) * 0.05)
    w2 = torch.nn.Parameter(torch.randn(72, K, device=cuda) * 0.05)
    b1 = torch.nn.Parameter(torch.randn(N - 72, device=cuda))
    b2 = torch.nn.Parameter(torch.randn(72, device=cuda))
    x = torch.randn(4, M // 4, K, device=cuda).to(dtype).requires_grad_()
    y = ops.linear(x, (w1, w2), (b1, b2), act="gelu")
    g = torch.randn_like(y)
    y.backward(g)
    xr = x.detach().double().requires_grad_()
    W = torch.cat([w1, w2]).detach().double().requires_grad_()
    bb = torch.cat([b1, b2]).detach().double().requires_grad_()
    yr = F.gelu(xr @ W.t() + bb)
    yr.backward(g.double())
    tol = 2e-5 if dtype == torch.float32 else 2e-2
    assert rel(y, yr) < tol
    assert rel(x.grad, xr.grad) < tol
    assert rel(torch.cat([w1.grad, w2.grad]), W.grad) < tol
    assert rel(torch.cat([b1.grad, b2.grad]), bb.grad) < tol


def _ref_attention(q, k, v, pe, maxpos, key_pad, causal, scale):
    """multihead_attention.py:340-389 in fp64. q,k,v [B,H,T,64]."""
    B, H, Tq, _ = q.shape
    Tk = k.shape[2]
    s = torch.einsum("bhic,bhjc->bhij", q * scale, k)
    if pe is not None:
        i = torch.arange(Tq, device=q.device)[:, None]; j = torch.arange(Tk, device=q.device)[None, :]
        idx = (i - j).clamp(-maxpos, maxpos - 1) + maxpos
        pos = pe[idx]  # [Tq,Tk,64]
        s = s + torch.einsum("bhic,ijc->bhij", q * scale, pos)
    if causal:
        s = s + torch.triu(torch.full((Tq, Tk), float("-inf"), device=q.device, dtype=s.dtype), 1)
    if key_pad is not None:
        s = s.masked_fill(key_pad[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    return torch.einsum("bhij,bhjc->bhic", p, v), p


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("case", ["self_rpe", "self_rpe_clip", "self_causal", "cross_probs"])
def test_attention(cuda, dtype, case):
    from speecht5_b200 import ops
    ops.RT.dtype = dtype
    torch.manual_seed(0)
    B, H = 2, 3
    d = H * 64
    maxpos = 160 if case != "self_rpe_clip" else 8
    Tq = 45 if case != "self_rpe_clip" else 37
    Tk = Tq if case.startswith("self") else 29
    lens = torch.tensor([Tk, Tk - 7], device=cuda)
    key_pad = torch.arange(Tk, device=cuda)[None, :] >= lens[:, None]
    pe = None
    if "rpe" in case:
        pe = torch.nn.Parameter(torch.randn(2 * maxpos, 64, device=cuda) * 0.3)
    if case.startswith("self"):
        qkv = (torch.randn(B, Tq, 3 * d, device=cuda) * 0.7).to(dtype).requires_grad_()
        out, probs = ops.attention(qkv, None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=0.125, pe_k=pe,
                                   maxpos=maxpos, key_pad=key_pad, causal=case == "self_causal")
        q, k, v = [t.reshape(B, Tq, H, 64).transpose(1, 2) for t in qkv.detach().double().split(d, dim=-1)]
    else:
        qb = (torch.randn(B, Tq, d, device=cuda) * 0.7).to(dtype).requires_grad_()
        kvb = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.7).to(dtype).requires_grad_()
        out, probs = ops.attention(qb, kvb, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=key_pad,
                                   return_probs=True)
        q = qb.detach().double().reshape(B, Tq, H, 64).transpose(1, 2)
        k, v = [t.reshape(B, Tk, H, 64).transpose(1, 2) for t in kvb.detach().double().split(d, dim=-1)]
    q, k, v = q.requires_grad_(), k.requires_grad_(), v.requires_grad_()
    per = pe.detach().double().requires_grad_() if pe is not None else None
    o_ref, p_ref = _ref_attention(q, k, v, per, maxpos, key_pad, case == "self_causal", 0.125)
    g = torch.randn(B, Tq, d, device=cuda)
    gp = torch.randn(B, H, Tq, Tk, device=cuda) if case == "cross_probs" else None
    loss = (out.float() * g).sum() + ((probs.float() * gp).sum() if gp is not None else 0)  # gp only with probs
    loss.backward()
    lr = (o_ref.transpose(1, 2).reshape(B, Tq, d) * g.double()).sum() + ((p_ref * gp.double()).sum() if gp is not None else 0)
    lr.backward()
    tol = 2e-5 if dtype == torch.float32 else 3e-2
    assert rel(out, o_ref.transpose(1, 2).reshape(B, Tq, d)) < tol
    if probs is not None:
        assert rel(probs, p_ref) < tol

    def flat(t):
        return t.transpose(1, 2).reshape(B, -1, d)
    if case.startswith("self"):
        gref = torch.cat([flat(q.grad), flat(k.grad), flat(v.grad)], -1)
        assert rel(qkv.grad, gref) < tol
        if pe is not None:
            assert rel(pe.grad, per.grad) < tol
    else:
        assert rel(qb.grad, flat(q.grad)) < tol
        assert rel(kvb.grad, torch.cat([flat(k.grad), flat(v.grad)], -1)) < tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_posenc_embedding(cuda, dtype):
    from speecht5_b200 import ops
    from speecht5_b200.models.modules.nets import sinusoid_table
    ops.RT.dtype = dtype
    torch.manual_seed(0)
    V, C, B, T = 81, 768, 3, 23
    emb = torch.nn.Parameter(torch.randn(V, C, device=cuda))
    alpha = torch.nn.Parameter(torch.tensor(1.3, device=cuda))
    tok = torch.randint(0, V, (B, T), device=cuda)
    tok[1, -4:] = 1
    pe = sinusoid_table(64, C, cuda)
    y = ops.scaled_posenc(pe, alpha, 0.0, tokens=tok, emb=emb, padding_idx=1)
    g = torch.randn(B, T, C, device=cuda)
    (y.float() * g).sum().backward()
    er, ar = emb.detach().double().requires_grad_(), alpha.detach().double().requires_grad_()
    yr = F.embedding(tok, er, padding_idx=1) + ar * pe[:T].double()
    (yr * g.double()).sum().backward()
    tol = 1e-5 if dtype == torch.float32 else 1e-2
    assert rel(y, yr) < tol and rel(emb.grad, er.grad) < tol
    # d(alpha) is a sum of B*T*C random-sign terms: compare on the scale of that random walk
    scale = (g.double() * pe[:T].double()).norm().item()
    assert abs(alpha.grad.item() - ar.grad.item()) < (1e-5 if dtype == torch.float32 else 2 ** -8) * scale


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_postnet_conv_bn(cuda, dtype):
    from speecht5_b200 import ops
    ops.RT.dtype = dtype
    torch.manual_seed(0)
    B, T, Cin, Cout = 3, 50, 80, 256
    conv = torch.nn.Conv1d(Cin, Cout, 5, padding=2, bias=False).to(cuda)
    bn = torch.nn.BatchNorm1d(Cout).to(cuda)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5); bn.bias.uniform_(-0.3, 0.3)
    x = torch.randn(B, T, Cin, device=cuda).to(dtype).requires_grad_()
    c = ops.conv1d_k5(x, conv.weight)
    y = ops.batch_norm_act(c, bn, training=True, act="tanh")
    g = torch.randn(B, T, Cout, device=cuda)
    (y.float() * g).sum().backward()
    convr = torch.nn.Conv1d(Cin, Cout, 5, padding=2, bias=False).to(cuda).double()
    bnr = torch.nn.BatchNorm1d(Cout).to(cuda).double()
    convr.load_state_dict(conv.state_dict())
    bnr.weight.data.copy_(bn.weight.data); bnr.bias.data.copy_(bn.bias.data)
    xr = x.detach().double().requires_grad_()
    yr = torch.tanh(bnr(convr(xr.transpose(1, 2)))).transpose(1, 2)
    (yr * g.double()).sum().backward()
    tol = 3e-5 if dtype == torch.float32 else 3e-2
    assert rel(y, yr) < tol
    assert rel(x.grad, xr.grad) < tol
    assert rel(conv.weight.grad, convr.weight.grad) < tol
    assert rel(bn.weight.grad, bnr.weight.grad) < tol and rel(bn.bias.grad, bnr.bias.grad) < tol
    stol = 1e-3 if dtype == torch.float32 else 2e-2
    assert rel(bn.running_mean, bnr.running_mean) < stol and rel(bn.running_var, bnr.running_var) < stol


def test_dropout_statistics_and_backward_mask(cuda):
    from speecht5_b200 import ops
    x = torch.ones(1 << 20, device=cuda, requires_grad=True)
    y = ops.dropout(x, 0.3)
    keep = (y != 0).float().mean().item()
    assert abs(keep - 0.7) < 5e-3
    assert abs(y.max().item() - 1 / 0.7) < 1e-5
    y.sum().backward()
    assert torch.equal(x.grad != 0, y != 0)


def test_adam_and_gradnorm(cuda):
    from speecht5_b200 import kernels as K
    torch.manual_seed(0)
    n = 100003
    p = torch.randn(n, device=cuda); g = torch.randn(n, device=cuda) * 3
    m = torch.zeros(n, device=cuda); v = torch.zeros(n, device=cuda)
    pb = torch.empty(n, device=cuda, dtype=torch.bfloat16)
    nsq = torch.zeros(1, device=cuda)
    K.sumsq(g, nsq)
    assert abs(nsq.item() - (g.double() ** 2).sum().item()) / nsq.item() < 1e-5
    pr, mr, vr = p.double().clone(), m.double().clone(), v.double().clone()
    lr, b1, b2, eps, max_norm = 1e-3, 0.9, 0.98, 1e-8, 25.0
    for step in (1, 2, 3):
        K.adam_step(p, g, m, v, pb, lr, b1, b2, eps, 0.0, step, nsq, max_norm, 0.5)
        gn = math.sqrt((g.double() ** 2).sum().item()) * 0.5
        gg = g.double() * 0.5 * min(1.0, max_norm / (gn + 1e-6))
        mr = b1 * mr + (1 - b1) * gg
        vr = b2 * vr + (1 - b2) * gg * gg
        pr = pr - lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step) * mr / (vr.sqrt() + eps)
    assert rel(p, pr) < 1e-5
    assert rel(pb.float(), pr) < 5e-3


@pytest.mark.parametrize("case", ["self_rpe", "cross"])
def test_tensor_core_attention_matches_row_kernels_with_dropout(cuda, case):
    """Same (seed, offset) => same Philox dropout mask in both implementations; outputs and gradients must agree."""
    from speecht5_b200 import ops
    ops.RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    B, H, Tq = 2, 4, 150
    d = H * 64
    Tk = Tq if case == "self_rpe" else 70
    lens = torch.tensor([Tk, Tk - 9], device=cuda)
    key_pad = torch.arange(Tk, device=cuda)[None, :] >= lens[:, None]
    pe = torch.nn.Parameter(torch.randn(320, 64, device=cuda) * 0.3) if case == "self_rpe" else None
    base_q = (torch.randn(B, Tq, (3 if case == "self_rpe" else 1) * d, device=cuda) * 0.7).to(torch.bfloat16)
    base_kv = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.7).to(torch.bfloat16)
    g = torch.randn(B, Tq, d, device=cuda).to(torch.bfloat16)
    res = []
    # (tensor core, fused): fused wgmma kernels / unfused tensor-core path (batched GEMMs + row kernels: the fallback
    # for clipped relative positions and long sequences) / exact row kernels.
    modes = [(True, True), (True, False), (False, True)]
    for tc, fused in modes:
        ops.RT.attn_tensor_core = tc
        ops.RT.attn_fused = fused
        ops.RT.manual_seed(5)
        qb = base_q.clone().requires_grad_()
        kvb = base_kv.clone().requires_grad_() if case == "cross" else None
        if pe is not None:
            pe.grad = None
        if case == "self_rpe":
            out, _ = ops.attention(qb, None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=0.125, pe_k=pe, maxpos=160,
                                   key_pad=key_pad, drop_p=0.2)
        else:
            out, _ = ops.attention(qb, kvb, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=key_pad,
                                   drop_p=0.2, return_probs=True)
        out.backward(g)
        res.append((out.detach(), qb.grad, kvb.grad if kvb is not None else None,
                    pe.grad.clone() if pe is not None else None))
    ops.RT.attn_tensor_core = True
    ops.RT.attn_fused = True
    for other in res[:-1]:
        for a, b in zip(other, res[-1]):
            if a is not None:
                assert rel(a, b) < 3e-2


@pytest.mark.parametrize("case", ["causal_313", "cross_313x160_probs", "self_64", "causal_130"])
def test_fused_attention_forward_and_backward(cuda, case):
    """Single-launch wgmma attention (attention_flash.cu) against the fp64 statement of multihead_attention.py."""
    from speecht5_b200 import ops
    ops.RT.dtype = torch.bfloat16
    ops.RT.attn_fused = True
    torch.manual_seed(1)
    B, H = 2, 3
    d = H * 64
    causal = case.startswith("causal")
    Tq = {"causal_313": 313, "cross_313x160_probs": 313, "self_64": 64, "causal_130": 130}[case]
    Tk = 160 if case.startswith("cross") else Tq
    lens = torch.tensor([Tk, max(1, Tk - 23)], device=cuda)
    key_pad = torch.arange(Tk, device=cuda)[None, :] >= lens[:, None]
    if case.startswith("cross"):
        qb = (torch.randn(B, Tq, d, device=cuda) * 0.8).to(torch.bfloat16).requires_grad_()
        kvb = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.8).to(torch.bfloat16).requires_grad_()
        out, probs = ops.attention(qb, kvb, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=key_pad,
                                   return_probs=True)
        q = qb.detach().double().reshape(B, Tq, H, 64).transpose(1, 2)
        k, v = [t.reshape(B, Tk, H, 64).transpose(1, 2) for t in kvb.detach().double().split(d, dim=-1)]
    else:
        qkv = (torch.randn(B, Tq, 3 * d, device=cuda) * 0.8).to(torch.bfloat16).requires_grad_()
        out, probs = ops.attention(qkv, None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=0.125, key_pad=key_pad,
                                   causal=causal)
        q, k, v = [t.reshape(B, Tq, H, 64).transpose(1, 2) for t in qkv.detach().double().split(d, dim=-1)]
    q, k, v = q.requires_grad_(), k.requires_grad_(), v.requires_grad_()
    o_ref, p_ref = _ref_attention(q, k, v, None, 0, key_pad, causal, 0.125)
    assert rel(out, o_ref.transpose(1, 2).reshape(B, Tq, d)) < 1.5e-2
    if probs is not None:  # self-attention with the fused backward keeps the probabilities on chip
        assert rel(probs, p_ref) < 1.5e-2
    g = torch.randn(B, Tq, d, device=cuda)
    (out.float() * g).sum().backward()
    (o_ref.transpose(1, 2).reshape(B, Tq, d) * g.double()).sum().backward()

    def flat(t):
        return t.transpose(1, 2).reshape(B, -1, d)
    if case.startswith("cross"):
        assert rel(qb.grad, flat(q.grad)) < 3e-2
        assert rel(kvb.grad, torch.cat([flat(k.grad), flat(v.grad)], -1)) < 3e-2
    else:
        assert rel(qkv.grad, torch.cat([flat(q.grad), flat(k.grad), flat(v.grad)], -1)) < 3e-2


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_conv0_groupnorm_gelu_against_the_oracle_layer(cuda, dtype):
    """csrc/conv_frontend.cu vs layer 0 of oracle ConvFeatureExtractionModel (mode "default"): forward activations and
    the gradients of the conv weight and the GroupNorm affine, ragged T (last block partial)."""
    from oracle.speecht5_oracle_asr import ConvFeatureExtractionModel
    from speecht5_b200 import kernels as K
    torch.manual_seed(3)
    B, n = 3, 5 * 700 + 10 + 3
    fe = ConvFeatureExtractionModel([(512, 10, 5)], mode="default").double()
    with torch.no_grad():
        fe.conv_layers[0][2].weight.add_(0.1 * torch.randn(512, dtype=torch.float64))
        fe.conv_layers[0][2].bias.add_(0.1 * torch.randn(512, dtype=torch.float64))
    wave = torch.randn(B, n, dtype=torch.float64) * 0.5 + 0.1
    y_ref = fe(wave).transpose(1, 2)  # [B, T0, C]
    T0 = y_ref.shape[1]
    assert T0 == (n - 10) // 5 + 1 and T0 % 128 != 0
    dy = torch.randn_like(y_ref)
    y_ref.backward(dy)
    conv, gn = fe.conv_layers[0][0], fe.conv_layers[0][2]
    w = conv.weight.detach().float().reshape(512, 10).contiguous().to(cuda)
    gamma, beta = gn.weight.detach().float().to(cuda), gn.bias.detach().float().to(cuda)
    wv = wave.float().to(cuda)
    y = torch.empty(B, T0, 512, device=cuda, dtype=dtype)
    mean = torch.empty(B, 512, device=cuda)
    rstd = torch.empty(B, 512, device=cuda)
    K.conv0_gn_gelu_fwd(wv, w, gamma, beta, y, mean, rstd, 5, gn.eps, "gelu")
    tol = 2e-5 if dtype == torch.float32 else 1e-2
    assert rel(y.cpu(), y_ref) < tol
    dw = torch.zeros(512, 10, device=cuda)
    dg = torch.zeros(512, device=cuda)
    db = torch.zeros(512, device=cuda)
    K.conv0_gn_gelu_bwd(dy.to(cuda).to(dtype).contiguous(), wv, w, gamma, beta, mean, rstd, dw, dg, db, 5, "gelu")
    assert rel(dw.cpu(), conv.weight.grad.reshape(512, 10)) < tol
    assert rel(dg.cpu(), gn.weight.grad) < tol
    assert rel(db.cpu(), gn.bias.grad) < tol


@pytest.mark.parametrize("case", ["rpe_199", "rpe_499_pad", "rpe_781", "rpe_small_table_37", "causal_500", "self_400_pad",
                                  "cross_160x499_probs", "cross_313x160_flash_probs_extdP"])
def test_streaming_attention_any_length(cuda, case):
    """attention_flash.cu (two sweeps over 128-key blocks, clipped relative positions) + the fused backward, against the
    fp64 statement of multihead_attention.py:340-389 / encoder.py:40-59 at the lengths SURVEY section 7 names (199, 499,
    781) -- padding, clipping at both table ends, a table smaller than one window, causal, returned probabilities with an
    external gradient on them."""
    from speecht5_b200 import ops
    ops.RT.dtype = torch.bfloat16
    ops.RT.attn_fused = ops.RT.attn_fused_bwd = ops.RT.attn_tensor_core = True
    keep = ops.RT.attn_flash
    ops.RT.attn_flash = "all"
    try:
        torch.manual_seed(2)
        B, H = 2, 2
        d = H * 64
        cfgs = {"rpe_199": (199, 199, 160, False), "rpe_499_pad": (499, 499, 160, False), "rpe_781": (781, 781, 160, False),
                "rpe_small_table_37": (37, 37, 8, False), "causal_500": (500, 500, 0, True),
                "self_400_pad": (400, 400, 0, False), "cross_160x499_probs": (160, 499, 0, False),
                "cross_313x160_flash_probs_extdP": (313, 160, 0, False)}
        Tq, Tk, maxpos, causal = cfgs[case]
        cross = case.startswith("cross")
        lens = torch.tensor([Tk, max(1, Tk - 37)], device=cuda)
        key_pad = torch.arange(Tk, device=cuda)[None, :] >= lens[:, None] if "causal" not in case else None
        pe = torch.nn.Parameter(torch.randn(2 * maxpos, 64, device=cuda) * 0.3) if maxpos else None
        if cross:
            qb = (torch.randn(B, Tq, d, device=cuda) * 0.8).to(torch.bfloat16).requires_grad_()
            kvb = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.8).to(torch.bfloat16).requires_grad_()
            out, probs = ops.attention(qb, kvb, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=key_pad,
                                       return_probs=True)
            q = qb.detach().double().reshape(B, Tq, H, 64).transpose(1, 2)
            k, v = [t.reshape(B, Tk, H, 64).transpose(1, 2) for t in kvb.detach().double().split(d, dim=-1)]
        else:
            qkv = (torch.randn(B, Tq, 3 * d, device=cuda) * 0.8).to(torch.bfloat16).requires_grad_()
            out, probs = ops.attention(qkv, None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=0.125, key_pad=key_pad,
                                       causal=causal, pe_k=pe, maxpos=maxpos)
            q, k, v = [t.reshape(B, Tq, H, 64).transpose(1, 2) for t in qkv.detach().double().split(d, dim=-1)]
        q, k, v = q.requires_grad_(), k.requires_grad_(), v.requires_grad_()
        # the kernel sees the bf16 copy of the table
        per = pe.detach().to(torch.bfloat16).double().requires_grad_() if pe is not None else None
        o_ref, p_ref = _ref_attention(q, k, v, per, maxpos, key_pad, causal, 0.125)
        assert rel(out, o_ref.transpose(1, 2).reshape(B, Tq, d)) < 1.5e-2
        g = torch.randn(B, Tq, d, device=cuda)
        gp = None
        if cross:
            assert probs is not None and probs.dtype == torch.float32
            assert rel(probs, p_ref) < 1e-2
            if "extdP" in case:
                gp = torch.randn(B, H, Tq, Tk, device=cuda)
        else:
            assert probs is None
        ((out.float() * g).sum() + ((probs * gp).sum() if gp is not None else 0)).backward()
        ((o_ref.transpose(1, 2).reshape(B, Tq, d) * g.double()).sum()
         + ((p_ref * gp.double()).sum() if gp is not None else 0)).backward()

        def flat(t):
            return t.transpose(1, 2).reshape(B, -1, d)
        if cross:
            assert rel(qb.grad, flat(q.grad)) < 3e-2
            assert rel(kvb.grad, torch.cat([flat(k.grad), flat(v.grad)], -1)) < 3e-2
        else:
            assert rel(qkv.grad, torch.cat([flat(q.grad), flat(k.grad), flat(v.grad)], -1)) < 3e-2
            if pe is not None:
                assert rel(pe.grad, per.grad) < 3e-2
    finally:
        ops.RT.attn_flash = keep


def test_streaming_attention_dropout_matches_row_kernels(cuda):
    """Same (seed, offset) => the same Philox mask in attention_flash.cu as in the exact row kernels, forward and (through
    the sign bits of the saved exponentials) backward."""
    from speecht5_b200 import ops
    ops.RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    B, H, T = 2, 2, 400
    d = H * 64
    base = (torch.randn(B, T, 3 * d, device=cuda) * 0.7).to(torch.bfloat16)
    g = torch.randn(B, T, d, device=cuda).to(torch.bfloat16)
    res = []
    for tc in (True, False):
        ops.RT.attn_tensor_core = tc
        ops.RT.manual_seed(7)
        qb = base.clone().requires_grad_()
        out, _ = ops.attention(qb, None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=0.125, causal=True, drop_p=0.2)
        out.backward(g)
        res.append((out.detach(), qb.grad))
    ops.RT.attn_tensor_core = True
    assert rel(res[0][0], res[1][0]) < 3e-2
    assert rel(res[0][1], res[1][1]) < 3e-2


@pytest.mark.parametrize("shape", [(768, 768, 10016, 8), (3072, 768, 5120, 2), (2304, 768, 5120, 2), (256, 200, 1024, 2),
                                   (768, 3072, 5120, 1)])
def test_weight_gradient_split_k_with_l2_reduce(cuda, shape):
    """accumulate = 2: dW += gy^T x with the contraction split over the batch dimension, every partial product added to
    the SAME fp32 output by a TMA reduce (cp.reduce.async.bulk.tensor .add) on 256 x 256 CTA-pair tiles -- against an
    fp64 product of the same bf16 operands, on top of a non-zero gradient buffer (fairseq accumulates micro-batches)."""
    from speecht5_b200 import kernels as K
    n_out, n_in, M, S = shape
    torch.manual_seed(3)
    gy = (torch.randn(M, n_out, device=cuda) * 0.5).to(torch.bfloat16)
    x = (torch.randn(M, n_in, device=cuda) * 0.5).to(torch.bfloat16)
    base = torch.randn(n_out, n_in, device=cuda)
    out = base.clone()
    chunk = M // S
    K.gemm(gy, x, out, M=n_out, N=n_in, K=chunk, a_mn=True, a_ld=n_out, b_mn=True, b_ld=n_in, c_ld=n_in, nb1=S, nb2=1,
           a_bs=(chunk * n_out, 0), b_bs=(chunk * n_in, 0), c_bs=(0, 0), accumulate=2)
    ref = base.double() + gy.double().t() @ x.double()
    assert rel(out, ref) < 2e-5  # fp32 accumulation over 5-10 k products per element (measured 1e-6 .. 6e-6)
    # and the same through the op the layers call, into a registered gradient view
    from speecht5_b200 import ops
    tgt = base.clone()
    ops.wgrad_mm((gy, None), n_out, (x, None), n_in, n_out, n_in, M, target=tgt)
    assert rel(tgt, ref) < 2e-5


def test_cross_attention_backward_with_a_gradient_on_two_heads_only(cuda):
    """RT.probs_grad_heads = n (set by the trainer from the guided-attention criterion): the external gradient on the
    returned probabilities is read for the first n heads only -- same result as the dense path when it is zero elsewhere."""
    from speecht5_b200 import ops
    ops.RT.dtype = torch.bfloat16
    torch.manual_seed(4)
    B, H, Tq, Tk = 2, 4, 200, 150
    d = H * 64
    base_q = (torch.randn(B, Tq, d, device=cuda) * 0.8).to(torch.bfloat16)
    base_kv = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.8).to(torch.bfloat16)
    g = torch.randn(B, Tq, d, device=cuda).to(torch.bfloat16)
    gp = torch.zeros(B, H, Tq, Tk, device=cuda)
    gp[:, :2] = torch.randn(B, 2, Tq, Tk, device=cuda)
    res = []
    for hint in (0, 2):
        ops.RT.probs_grad_heads = hint
        qb, kvb = base_q.clone().requires_grad_(), base_kv.clone().requires_grad_()
        out, probs = ops.attention(qb, kvb, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, return_probs=True)
        torch.autograd.backward([out, probs], [g, gp])
        res.append((qb.grad, kvb.grad))
    ops.RT.probs_grad_heads = 0
    # (the guided heads' row constant is summed in two launches -- dO.O on the vector path, sum P dP_ext per warp -- so
    #  its fp32 order differs from the all-heads form: an occasional last-bit flip of a bf16 gradient)
    assert rel(res[1][0], res[0][0]) < 2e-4 and rel(res[1][1], res[0][1]) < 2e-4


@pytest.mark.parametrize("r,B,L,D,Ly", [(2, 5, 62, 80, 64), (1, 3, 33, 80, 33), (2, 4, 20, 30, 27)])
def test_fused_tts_criterion_kernels_against_the_torch_formulation(cuda, r, B, L, D, Ly):
    """csrc/criterion.cu through TacotronLossFn: (l1, l2, bce) and their gradients vs Tacotron2Loss (the broadcast torch
    statement of text_to_speech_loss.py:217-345) in fp64 -- ragged lengths, lengths that are not multiples of r, targets
    longer than the output, the forced stop label of the last valid frame, odd feature widths (scalar path)."""
    from speecht5_b200.criterions.text_to_speech_loss import Tacotron2Loss, TacotronLossFn
    torch.manual_seed(3)
    after = torch.randn(B, L, D, device=cuda).requires_grad_()
    before = torch.randn(B, L, D, device=cuda).requires_grad_()
    logits = (torch.randn(B, L, device=cuda) * 2).requires_grad_()
    ys = torch.randn(B, Ly, D, device=cuda)
    olens = torch.tensor([L, L - 1, max(r, L // 2), r, L - 3][:B], device=cuda)
    labels = torch.zeros(B, Ly, device=cuda)
    for b in range(B):
        labels[b, int(olens[b]) - 1:] = 1.0
    got = TacotronLossFn.apply(after, before, logits, ys, labels, olens, r, 5.0)
    w = torch.tensor([1.0, 0.3, 0.7], device=cuda)
    (got * w).sum().backward()
    a64, b64, l64 = (t.detach().double().requires_grad_() for t in (after, before, logits))
    ol = olens - olens % r
    y64, lab64 = ys[:, :L].double(), labels[:, :L].double().clone()
    if r > 1:
        lab64 = torch.scatter(lab64, 1, (ol - 1).unsqueeze(1), 1.0)
    want = torch.stack(Tacotron2Loss(bce_pos_weight=5.0).to(cuda).double()(a64, b64, l64, y64, lab64, ol))
    (want * w.double()).sum().backward()
    assert rel(got, want) < 1e-5
    assert rel(after.grad, a64.grad) < 1e-5 and rel(before.grad, b64.grad) < 1e-5 and rel(logits.grad, l64.grad) < 1e-5
    assert float(after.grad[1, L - 1].abs().max()) == 0.0  # (a masked frame)


@pytest.mark.parametrize("T_in,sparse", [(160, True), (160, False), (37, False)])
def test_fused_guided_attention_kernels_against_the_torch_formulation(cuda, T_in, sparse):
    """GuidedAttnFn vs GuidedMultiHeadAttentionLoss over torch.cat of the head slices (text_to_speech_loss.py:370-427):
    several layers read in place, a row pitch that differs from T_in, and the backward with / without touching the heads
    the attention backward never reads."""
    from speecht5_b200.criterions.text_to_speech_loss import GuidedAttnFn, GuidedMultiHeadAttentionLoss
    torch.manual_seed(4)
    B, H, T_out, heads, r = 3, 12, 41, 2, 2
    p_ld = (T_in + 7) // 8 * 8
    bufs = [torch.rand(B, H, T_out, p_ld, device=cuda) for _ in range(3)]
    atts = [(b[..., :T_in] if p_ld != T_in else b).requires_grad_() for b in bufs]
    if sparse:
        for a in atts:
            a._st5_ext_heads = heads
    ilens = torch.tensor([T_in, T_in - 5, 9], device=cuda)
    olens = torch.tensor([2 * T_out, 2 * T_out - 3, 30], device=cuda)
    got = GuidedAttnFn.apply(ilens, olens, r, heads, 0.4, 1.0, *atts)
    grads = torch.autograd.grad(got * 3.0, atts)
    ref_in = [a.detach().double().requires_grad_() for a in atts]
    want = GuidedMultiHeadAttentionLoss(0.4, 1.0)(torch.cat([a[:, :heads] for a in ref_in], 1), ilens,
                                                  torch.div(olens, r, rounding_mode="floor"))
    ref_grads = torch.autograd.grad(want * 3.0, ref_in)
    assert abs(got.item() - want.item()) < 1e-5 * abs(want.item())
    for g, rg in zip(grads, ref_grads):
        assert rel(g[:, :heads], rg[:, :heads]) < 1e-5
        if not sparse:
            assert float(g[:, heads:].abs().max()) == 0.0


@pytest.mark.parametrize("Tq,Tk", [(313, 160), (200, 499)])
def test_returned_probabilities_for_the_first_heads_only(cuda, Tq, Tk):
    """RT.probs_read_heads (set by B200Trainer for the duration of an update: the guided-attention loss is the only
    reader of the returned cross-attention maps, text_to_speech_loss.py:210-212): the fused (Tk <= 320) and the
    streaming forward write the probabilities of heads < n only -- same output, same first-n maps, same gradients."""
    from speecht5_b200 import ops
    from speecht5_b200.ops import RT
    RT.dtype = torch.bfloat16
    torch.manual_seed(2)
    B, H, d = 2, 12, 768
    q = (torch.randn(B, Tq, d, device=cuda) * 0.5).bfloat16()
    kv = (torch.randn(B, Tk, 2 * d, device=cuda) * 0.5).bfloat16()
    pad = torch.zeros(B, Tk, dtype=torch.bool, device=cuda)
    pad[1, Tk - 9:] = True
    res = []
    for n in (0, 2):
        RT.probs_read_heads = RT.probs_grad_heads = n
        try:
            qq, kk = q.clone().requires_grad_(), kv.clone().requires_grad_()
            out, probs = ops.attention(qq, kk, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=pad, return_probs=True)
            g = torch.zeros_like(probs)
            g[:, :2] = torch.randn(B, 2, Tq, Tk, device=cuda, generator=torch.Generator(device=cuda).manual_seed(9))
            (out.float().square().sum() + (probs[:, :2] * g[:, :2]).sum()).backward()
            res.append((out.detach().clone(), probs.detach()[:, :2].clone(), qq.grad.clone(), kk.grad.clone(), g))
        finally:
            RT.probs_read_heads = RT.probs_grad_heads = 0
    (o0, p0, dq0, dk0, g0), (o1, p1, dq1, dk1, g1) = res
    assert torch.equal(o0, o1) and torch.equal(p0, p1)
    assert (p1[0].sum(-1) - 1).abs().max() < 1e-3
    assert rel(dq1, dq0) < 2e-4 and rel(dk1, dk0) < 2e-4  # (row constants summed in a different fp32 order)

"""The window-GEMM convolution compositions run on NaN-filled buffers and checked elementwise against tests/conv_ref.py.
tests/test_conv_contract_gpu.py runs them on the device; tests/test_conv_ref_cpu.py runs them on the GEMM emulator,
with and without injected faults.

While a composition runs, torch.empty / torch.empty_like hand out NaN-filled floating tensors (`nan_empty`), so an
element that no GEMM or phase writes cannot pass by luck; the zero-padding buffers come from torch.zeros and are read
by design. Every runner returns {name: largest err / bound} and raises on the first element out of bound."""
import contextlib
import math

import torch

import conv_ref as C

NAN = float("nan")
BF16, F32 = torch.bfloat16, torch.float32


@contextlib.contextmanager
def nan_empty():
    empty, empty_like = torch.empty, torch.empty_like

    def _empty(*a, **kw):
        t = empty(*a, **kw)
        return t.fill_(NAN) if t.is_floating_point() else t

    def _empty_like(*a, **kw):
        t = empty_like(*a, **kw)
        return t.fill_(NAN) if t.is_floating_point() else t
    torch.empty, torch.empty_like = _empty, _empty_like
    try:
        yield
    finally:
        torch.empty, torch.empty_like = empty, empty_like


@contextlib.contextmanager
def numeric_mode(dtype):
    """RT.dtype for the call, with the weight shadows re-cast before and after (ids of fresh weights get reused)."""
    from speecht5_b200.ops import RT
    old = RT.dtype
    RT.dtype = dtype
    RT.invalidate_shadows()
    try:
        yield RT
    finally:
        RT.dtype = old
        RT.invalidate_shadows()


def mode_name(dtype):
    return "bf16" if dtype == BF16 else "fp32"


def _rand(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, dtype=torch.float64).float() * scale


def _check(out, name, got, ref, bound):
    out[name] = max(out.get(name, 0.0), C.check(name, got, ref, bound))


def _dev_act(act, dtype):
    """The activation the composition asks the epilogue for (ops._resolve_act)."""
    return None if act is None else ("gelu_tanh" if dtype == BF16 else "gelu")


# ============================================================================================ post-net Conv1d k5
def postnet(dev, Cin, Cout, B, T, dtype, seed=0):
    """ops.conv1d_k5 forward, dx and dW. Returns (ratios, info) with the weight-gradient split the backward took."""
    from speecht5_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    x = _rand(gen, B, T, Cin, scale=0.8).to(dtype).to(dev).requires_grad_()
    w = _rand(gen, Cout, Cin, 5, scale=(5 * Cin) ** -0.5).to(dev).requires_grad_()
    dy = _rand(gen, B, T, Cout).to(dtype).to(dev)
    Kd = B * (T + 4) - 4
    S, chunk = ops._conv_wgrad_split(Cout, 5 * Cin, Kd)
    with numeric_mode(dtype) as RT, nan_empty():
        split = dtype == BF16 and RT.wgrad_splitk and S > 1 and Cout % 8 == 0 and Cin % 8 == 0
        y = ops.conv1d_k5(x, w)
        y.backward(dy)
    out, m = {}, f"postnet {mode_name(dtype)}"
    u = C.unit(dtype)
    conv = C.Conv(lambda a, b: C.conv1d_cl(a, b, padding=2), x.detach(), C.weight_as_read(w.detach(), dtype))
    acc, mag = conv.forward()
    e = C.epilogue(acc, C.product_bound(mag, 5 * Cin, dtype), u_out=u)
    _check(out, f"{m} y", y.detach(), e["y"], e["e_y"])
    g = dy.to(torch.float64)
    b = C.grad_bounds(conv, g, torch.zeros_like(g), K_dx=5 * Cout, K_dw=Kd, dtype=dtype, u_dx=u,
                      dw_sum_terms=S if split else 0)
    _check(out, f"{m} dx", x.grad, b["dx"], b["e_dx"])
    _check(out, f"{m} dW", w.grad, b["dw"], b["e_dw"])
    return out, dict(S=S, chunk=chunk, Kd=Kd, split=split)


# ============================================================================================ strided front end
def strided(dev, k, s, Cin, Cout, B, T, act, dtype, seed=0, backward=True):
    """frontend.StridedConvGeluFn forward (and the stored pre-activation), dx and dW; frames that no output window
    covers must get an exactly zero input gradient."""
    from speecht5_b200 import frontend
    gen = torch.Generator().manual_seed(seed)
    To = (T - k) // s + 1
    x = _rand(gen, B, T, Cin, scale=0.8).to(dtype).to(dev).requires_grad_(backward)
    w = _rand(gen, Cout, Cin, k, scale=(k * Cin) ** -0.5).to(dev).requires_grad_(backward)
    dy = _rand(gen, B, To, Cout).to(dtype).to(dev)
    dact = _dev_act(act, dtype)
    with numeric_mode(dtype), nan_empty():
        y = frontend.StridedConvGeluFn.apply(x, w, s, act)
        if backward:
            pre_saved = y.grad_fn.saved_tensors[1]
            y.backward(dy)
    out, m = {}, f"strided {mode_name(dtype)}"
    u = C.unit(dtype)
    conv = C.Conv(lambda a, b: C.conv1d_cl(a, b, stride=s), x.detach(), C.weight_as_read(w.detach(), dtype))
    acc, mag = conv.forward()
    e = C.epilogue(acc, C.product_bound(mag, k * Cin, dtype), u_out=u, act=dact)
    _check(out, f"{m} y", y.detach(), e["y"], e["e_y"])
    if not backward:
        return out
    if dact is not None:
        _check(out, f"{m} pre", pre_saved, e["pre"], e["e_pre"])
    g, e_g = C.act_grad_input(dy, pre_saved, dact, u)
    b = C.grad_bounds(conv, g, e_g, K_dx=-(-k // s) * Cout, K_dw=To, dtype=dtype, u_dx=u, dw_sum_terms=B)
    _check(out, f"{m} dx", x.grad, b["dx"], b["e_dx"])
    _check(out, f"{m} dW", w.grad, b["dw"], b["e_dw"])
    read = torch.zeros(T, dtype=torch.bool)
    for o in range(To):
        read[o * s:o * s + k] = True
    unread = x.grad[:, ~read.to(dev)]
    assert bool((unread == 0).all()), f"{m}: frames no output reads have a non-zero input gradient"
    return out


# ============================================================================================ positional conv
def posconv(dev, Cc, G, k, B, T, dtype, seed=0):
    """frontend.GroupedPosConvFn: y = x + GELU(SamePad(grouped Conv1d) + bias); forward, pre, dx, dW, dbias."""
    from speecht5_b200 import frontend
    gen = torch.Generator().manual_seed(seed)
    cg = Cc // G
    x = _rand(gen, B, T, Cc, scale=0.8).to(dtype).to(dev).requires_grad_()
    w = _rand(gen, Cc, cg, k, scale=(k * cg) ** -0.5).to(dev).requires_grad_()
    bias = _rand(gen, Cc, scale=0.1).to(dev).requires_grad_()
    dy = _rand(gen, B, T, Cc).to(dtype).to(dev)
    dact = _dev_act("gelu", dtype)
    with numeric_mode(dtype), nan_empty():
        y = frontend.GroupedPosConvFn.apply(x, w, bias, G)
        pre_saved = y.grad_fn.saved_tensors[1]
        y.backward(dy)
    out, m = {}, f"posconv {mode_name(dtype)}"
    u = C.unit(dtype)
    conv = C.Conv(lambda a, b: C.conv1d_cl(a, b, padding=k // 2, groups=G, length=T), x.detach(),
                  C.weight_as_read(w.detach(), dtype))
    acc, mag = conv.forward()
    e = C.epilogue(acc, C.product_bound(mag, k * cg, dtype), u_out=u, bias=bias.detach(), act=dact,
                   residual=x.detach())
    _check(out, f"{m} y", y.detach(), e["y"], e["e_y"])
    _check(out, f"{m} pre", pre_saved, e["pre"], e["e_pre"])
    g, e_g = C.act_grad_input(dy, pre_saved, dact, u)
    b = C.grad_bounds(conv, g, e_g, K_dx=k * cg, K_dw=B * (T + k) - (k - 1), dtype=dtype, u_dx=u, dx_extra=dy)
    _check(out, f"{m} dx", x.grad, b["dx"], b["e_dx"])
    _check(out, f"{m} dW", w.grad, b["dw"], b["e_dw"])
    db, e_db = C.colsum_bound(g, e_g, (0, 1))
    _check(out, f"{m} dbias", bias.grad, db, e_db)
    return out


# ============================================================================================ HiFi-GAN
def hifi_same(dev, Cin, Cout, k, d, B, T, *, slope=None, residual=False, act=None, out_dtype=BF16, out_buffer=True,
              seed=0, name="same"):
    """vocoder._conv_same (bf16 operands, inference): leaky-ReLU + zero padding + de-interleave by st5_lrelu_pad, d
    phase GEMMs written back at pitch d Cout, bias / residual / act in the epilogue. out_buffer: pass a NaN `out=`."""
    from speecht5_b200 import vocoder
    gen = torch.Generator().manual_seed(seed)
    x = _rand(gen, B, T, Cin, scale=0.8).to(BF16).to(dev)
    w = _rand(gen, Cout, Cin, k, scale=(k * Cin) ** -0.5).to(dev)
    bias = _rand(gen, Cout, scale=0.1).to(dev)
    with nan_empty():
        conv = vocoder._Conv(w, bias, d)
        out = torch.full((B, T, Cout), NAN, dtype=out_dtype, device=dev) if out_buffer else None
        y = vocoder._conv_same(x, conv, out=out, act=act, residual=x if residual else None, pre_act_slope=slope)
    xh = C.lrelu_bf16(x, slope) if slope is not None else x.to(torch.float64)
    cv = C.Conv(lambda a, b: C.conv1d_cl(a, b, padding=(k * d - d) // 2, dilation=d), xh, C.weight_as_read(w, BF16))
    acc, mag = cv.forward()
    e = C.epilogue(acc, C.product_bound(mag, k * Cin, BF16), u_out=C.unit(out_dtype), bias=bias, act=act,
                   residual=x if residual else None)
    res = {}
    _check(res, f"hifigan {name}", y, e["y"], e["e_y"])
    return res


def hifi_transpose(dev, Cin, Cout, B, T, *, k=8, u=4, p=2, slope=0.1, seed=0, fault=None):
    """vocoder._conv_transpose: u phase GEMMs over the padded input at offset (fr + d0) Cin, written at pitch u Cout.
    fault(ct) may edit the phase table before the call (tests/test_conv_ref_cpu.py)."""
    from speecht5_b200 import vocoder
    gen = torch.Generator().manual_seed(seed)
    x = _rand(gen, B, T, Cin, scale=0.8).to(BF16).to(dev)
    w = _rand(gen, Cin, Cout, k, scale=(k // u * Cin) ** -0.5).to(dev)
    bias = _rand(gen, Cout, scale=0.1).to(dev)
    with nan_empty():
        ct = vocoder._ConvT(w, bias, u, p)
        if fault is not None:
            fault(ct)
        y = vocoder._conv_transpose(x, ct, pre_act_slope=slope)
    cv = C.Conv(lambda a, b: C.conv_transpose1d_cl(a, b, stride=u, padding=p), C.lrelu_bf16(x, slope),
                C.weight_as_read(w, BF16))
    acc, mag = cv.forward()
    e = C.epilogue(acc, C.product_bound(mag, ct.taps * Cin, BF16), u_out=C.U16, bias=bias)
    res = {}
    _check(res, "hifigan transpose", y, e["y"], e["e_y"])
    return res


def merge(report, ratios):
    for k_, v in ratios.items():
        report[k_] = max(report.get(k_, 0.0), v)


def margin(K, u_out, dtype):
    """How many times one product term (mag / sqrt(K)) exceeds the bound (module docstring of tests/conv_ref.py)."""
    b = C.C_ACC * C.U32 * K + (u_out if dtype == BF16 else C.SPLIT * math.sqrt(K))
    return 1.0 / b

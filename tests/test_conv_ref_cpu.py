"""CPU: the fp64 statements and bounds of tests/conv_ref.py. The statements are checked against torch's own
convolution modules and an explicit tap sum; the parity-mode split constant against real bf16 splits. Then the
compositions run on the GEMM emulator (tests/gemm_emulator.py) through tests/conv_cases.py: they pass the bounds as
they are, and fail them with each injected fault -- a dropped last k-block, a skipped split-K chunk, an input-gradient
phase read one row off and a transposed-conv tap offset off by one."""
import pytest
import torch
import torch.nn.functional as F

import conv_cases as CC
import conv_ref as C
import gemm_emulator

F64 = torch.float64
MODES = [torch.bfloat16, torch.float32]
MODE_IDS = ["bf16", "fp32"]


# ------------------------------------------------------------------------------------------------ statements
def _module_grads(mod, x, dy, length):
    """torch autograd of an nn module on channels-last x, output cut to `length` frames: (y, dx, dW)."""
    x = x.clone().requires_grad_()
    y = mod(x.transpose(1, 2))[..., :length].transpose(1, 2)
    y.backward(dy)
    return y.detach(), x.grad, mod.weight.grad


@pytest.mark.parametrize("case", ["postnet", "strided", "posconv", "dilated", "transpose"])
def test_statements_match_torch_modules(case):
    torch.manual_seed(0)
    B, T, Ci, Co = 2, 23, 6, 8
    x = torch.randn(B, T, Ci, dtype=F64)
    length = None
    if case == "postnet":
        mod, fn = torch.nn.Conv1d(Ci, Co, 5, padding=2, bias=False), lambda a, w: C.conv1d_cl(a, w, padding=2)
    elif case == "strided":
        mod, fn = torch.nn.Conv1d(Ci, Co, 5, stride=3, bias=False), lambda a, w: C.conv1d_cl(a, w, stride=3)
    elif case == "posconv":  # SamePad of an even kernel: the last frame dropped
        mod = torch.nn.Conv1d(Ci, Ci, 4, padding=2, groups=2, bias=False)
        fn, length = (lambda a, w: C.conv1d_cl(a, w, padding=2, groups=2, length=T)), T
    elif case == "dilated":
        mod, fn = torch.nn.Conv1d(Ci, Co, 7, dilation=3, padding=9, bias=False), \
            lambda a, w: C.conv1d_cl(a, w, padding=9, dilation=3)
    else:
        mod, fn = torch.nn.ConvTranspose1d(Ci, Co, 8, stride=4, padding=2, bias=False), \
            lambda a, w: C.conv_transpose1d_cl(a, w, stride=4, padding=2)
    mod = mod.double()
    with torch.no_grad():
        dy = torch.randn_like(mod(x.transpose(1, 2))[..., :length].transpose(1, 2))
    y, dx, dw = _module_grads(mod, x, dy, length)
    conv = C.Conv(fn, x, mod.weight.detach())
    got, mag = conv.forward()
    gx, gw = conv.vjp(dy)
    assert torch.allclose(got, y, rtol=1e-12, atol=1e-12)
    assert torch.allclose(gx, dx, rtol=1e-12, atol=1e-12) and torch.allclose(gw, dw, rtol=1e-12, atol=1e-12)
    assert bool((mag >= got.abs() - 1e-12).all())
    mx, mw = conv.vjp_mag(dy.abs())
    assert bool((mx >= gx.abs() - 1e-12).all()) and bool((mw >= gw.abs() - 1e-12).all())


def test_strided_dilated_statement_is_the_tap_sum():
    """y[b, t, co] = sum_j sum_ci x[b, s t + d j - pad, ci] w[co, ci, j] (zeros outside [0, T)), written as loops."""
    torch.manual_seed(1)
    B, T, Ci, Co, k, s, d, pad = 2, 19, 3, 4, 3, 2, 2, 2
    x, w = torch.randn(B, T, Ci, dtype=F64), torch.randn(Co, Ci, k, dtype=F64)
    got = C.conv1d_cl(x, w, stride=s, dilation=d, padding=pad)
    To = (T + 2 * pad - d * (k - 1) - 1) // s + 1
    want = torch.zeros(B, To, Co, dtype=F64)
    for t in range(To):
        for j in range(k):
            i = s * t + d * j - pad
            if 0 <= i < T:
                want[:, t] += x[:, i] @ w[:, :, j].T
    assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)


def test_parity_split_constant_bounds_the_dropped_terms():
    """|x w - (hi_x hi_w + hi_x lo_w + lo_x hi_w)| <= SPLIT |x w| for the bf16 splits st5_cast_bf16 makes, and SPLIT
    is not loose by more than a factor of a few."""
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1 << 20, generator=g) * torch.exp(torch.randn(1 << 20, generator=g) * 3)
    w = torch.randn(1 << 20, generator=g)

    def split(v):
        hi = v.to(torch.bfloat16)
        return hi.to(F64), (v - hi.float()).to(torch.bfloat16).to(F64)
    (xh, xl), (wh, wl) = split(x), split(w)
    exact = x.to(F64) * w.to(F64)
    drop = (exact - (xh * wh + xh * wl + xl * wh)).abs() / exact.abs()
    worst = float(drop.max())
    assert worst <= C.SPLIT and worst > C.SPLIT / 8, (worst, C.SPLIT)


def test_margins_stated_in_the_docstring():
    """The per-family factors by which one product term exceeds the bound (tests/conv_ref.py docstring)."""
    bf, fp = torch.bfloat16, torch.float32
    for K, lo_bf, lo_fp in ((400, 233, 770), (1280, 195, 349), (1024, 205, 409), (2560, 158, 210),
                            (6144, 102, 106), (8192, 85, 84)):
        assert round(CC.margin(K, C.U16, bf)) >= lo_bf and round(CC.margin(K, C.U16, fp)) >= lo_fp, K
    assert round(CC.margin(2112, 0.0, bf)) >= 496 and round(CC.margin(2112, 0.0, fp)) >= 243
    assert round(CC.margin(11 * 512, C.U16, bf)) >= 108


# ------------------------------------------------------------------------------------------------ compositions
class Faults:
    """st5_gemm_bf16 on the emulator with one injected defect; `hits` counts the launches it changed."""

    def __init__(self, monkeypatch, kind=None):
        gemm_emulator.install(monkeypatch)
        from speecht5_b200 import kernels as K
        self.base, self.kind, self.hits = K.gemm, kind, 0
        if kind is not None:
            monkeypatch.setattr(K, "gemm", self.gemm)

    def gemm(self, a, b, out, **kw):
        if self.kind == "drop_last_kblock" and kw["K"] > 64:
            kw["K"] = (kw["K"] - 1) // 64 * 64
            self.hits += 1
        elif self.kind == "skip_split_chunk" and int(kw.get("accumulate", 0)) == 2 and kw.get("nb1", 1) > 1:
            kw["nb1"] -= 1
            self.hits += 1
        elif self.kind == "phase_row_shift" and kw.get("c_ld") not in (None, kw["N"]) and not kw.get("a_mn"):
            a = a.reshape(-1)[kw["a_ld"]:]  # the phase reads its gradient windows one row late
            self.hits += 1
        return self.base(a, b, out, **kw)


def _fails(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
def test_postnet_on_the_emulator(monkeypatch, dtype):
    Faults(monkeypatch)
    for B, T in ((1, 1), (2, 9), (3, 350)):
        CC.postnet("cpu", 32, 24, B, T, dtype, seed=T)
    _, info = CC.postnet("cpu", 32, 32, 3, 350, dtype, seed=1)
    assert info["split"] == (dtype == torch.bfloat16) and info["S"] * info["chunk"] > info["Kd"]


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("act", ["gelu", None], ids=["gelu", "layer_norm"])
def test_strided_on_the_emulator(monkeypatch, dtype, act):
    Faults(monkeypatch)
    for k, s, T in ((3, 2, 3), (3, 2, 20), (2, 2, 21), (5, 3, 22), (4, 2, 19), (2, 3, 20)):
        CC.strided("cpu", k, s, 16, 24, 2, T, act, dtype, seed=T)


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
def test_positional_conv_on_the_emulator(monkeypatch, dtype):
    Faults(monkeypatch)
    for T in (1, 19, 40):
        CC.posconv("cpu", 32, 2, 8, 3, T, dtype, seed=T)


def test_hifigan_on_the_emulator(monkeypatch):
    Faults(monkeypatch)
    for k, d, T in ((3, 1, 1), (3, 5, 2), (7, 3, 37), (11, 5, 4)):
        CC.hifi_same("cpu", 16, 16, k, d, 2, T, slope=0.1, residual=True, seed=T)
    CC.hifi_same("cpu", 16, 1, 7, 1, 2, 13, slope=0.01, act="tanh", out_dtype=torch.float32)
    CC.hifi_same("cpu", 16, 32, 7, 1, 2, 13, out_buffer=False)
    CC.hifi_transpose("cpu", 16, 8, 2, 13)


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
def test_a_dropped_last_k_block_leaves_the_bounds(monkeypatch, dtype):
    for run in (lambda: CC.postnet("cpu", 32, 24, 2, 9, dtype),
                lambda: CC.strided("cpu", 3, 2, 32, 24, 2, 20, "gelu", dtype),
                lambda: CC.posconv("cpu", 32, 2, 8, 2, 19, dtype)):
        f = Faults(monkeypatch, "drop_last_kblock")
        assert _fails(run) and f.hits > 0


def test_a_skipped_split_k_chunk_leaves_the_bounds(monkeypatch):
    f = Faults(monkeypatch, "skip_split_chunk")
    r = {}
    assert _fails(lambda: r.update(CC.postnet("cpu", 32, 32, 3, 350, torch.bfloat16, seed=1)[0]))
    assert f.hits == 1


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
def test_an_input_gradient_phase_one_row_off_leaves_the_bounds(monkeypatch, dtype):
    f = Faults(monkeypatch, "phase_row_shift")
    assert _fails(lambda: CC.strided("cpu", 3, 2, 16, 24, 2, 20, None, dtype))
    assert f.hits > 0


def test_a_transposed_conv_tap_offset_off_by_one_leaves_the_bounds(monkeypatch):
    Faults(monkeypatch)

    def shift(ct):
        d0, nt, w, ld = ct.phases[0]
        ct.phases[0] = (d0 + 1, nt, w, ld)
    assert _fails(lambda: CC.hifi_transpose("cpu", 16, 8, 2, 13, fault=shift))

"""-m gpu: the waveform front-end (st5_conv0_gn_gelu_*, st5_conv0_ln_gelu_*) and decode-attention (st5_attn_decode_fwd)
entry points of include/speecht5_b200.h called through ctypes (speecht5_b200/_lib.py) against the fp64 statements of
tests/frontend_ref.py and tests/attention_ref.py with ELEMENTWISE bounds, on buffers laid out with NaN sentinels
everywhere the contract does not let a kernel read or write:
  - every output sits inside a NaN buffer with guard zones; scratch starts NaN; dw / dgamma / dbeta start non-zero;
  - waveform samples past (T0 - 1) S + K are NaN (never read);
  - decode: q / k / v live in fused q|k|v rows whose other column blocks are NaN, the K / V rows of masked keys and the
    rows [Tk, buffer) are NaN, and the gaps of an o_bs > H * 64 output are NaN.
Shapes reach the GroupNorm channel groups (C > 512 runs on grid.z), the chunk edges (T0 = 127 / 128 / 129), the
largest stride whose staged segment fits in 48 KiB, both LayerNorm backward instantiations (K <= 10 and K > 10), a
persistent grid larger than 2 x SMs, and the decode splits (Tk = 64 / 65, 128 / 129, thousands of keys). Every negative
return leaves every buffer bit-identical. The largest err / bound per entry point is printed at the end (run with -s)."""
import ctypes as ct
import math

import pytest
import torch

import attention_ref as A
import frontend_ref as R

pytestmark = pytest.mark.gpu

NAN = float("nan")
G = 64  # guard elements before and after every buffer
REPORT = {}
F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
ACTS = {"gelu": 2, "gelu_tanh": 4}
DT = {F32: 0, BF16: 1}
EPS = 1e-5


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per entry point:")
        for k in sorted(REPORT):
            print(f"  {k:44s} {REPORT[k]:.3g}")


def _lib():
    from speecht5_b200 import _lib as L
    return L.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def P(t):
    return None if t is None else ct.c_void_p(t.data_ptr())


class Buf:
    """n elements inside a NaN buffer with guard zones (`off` elements past the 16-byte aligned start)."""

    def __init__(self, n, dtype=F32, fill=None, off=0):
        self.flat = torch.full((2 * G + n + off,), NAN, dtype=dtype, device="cuda")
        self.lo, self.hi = G + off, G + off + n
        self.t = self.flat[self.lo:self.hi]
        if fill is not None:
            self.t.copy_(torch.as_tensor(fill).reshape(-1).to(dtype))

    def untouched(self, what):
        g = torch.cat([self.flat[:self.lo], self.flat[self.hi:]]).float()
        assert bool(torch.isnan(g).all()), f"{what}: guard zone written"

    def snapshot(self):
        return self.flat.clone()

    def same_as(self, snap):
        w = torch.int16 if self.flat.dtype == BF16 else torch.int32
        return bool(torch.equal(self.flat.view(w), snap.view(w)))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _f32(t):
    return t.float().double()


# ============================================================================================ conv0 inputs
def _wave(B, T0, K, S, kind, seed):
    """[B, n] fp32 with n = (T0 - 1) S + K + (S - 1): the last S - 1 samples are unread (NaN)."""
    used = (T0 - 1) * S + K
    n = used + S - 1
    g = _gen(seed)
    if kind == "rand":
        x = torch.randn(B, used, generator=g, dtype=F64) * 0.1
    elif kind == "const":          # zero variance: rstd = eps^-1/2
        x = torch.full((B, used), 0.3, dtype=F64)
    elif kind == "dc":             # a large DC offset under a small signal
        x = 100.0 + 0.01 * torch.randn(B, used, generator=g, dtype=F64)
    elif kind == "click":          # the first frame of every chunk far from its chunk's mean
        x = 0.01 * torch.randn(B, used, generator=g, dtype=F64)
        x[:, 0:used:128 * S] += 50.0
    elif kind == "silence":
        x = torch.zeros(B, used, dtype=F64)
    else:
        raise ValueError(kind)
    host = torch.full((B, n), NAN, dtype=F32)
    host[:, :used] = x.float()
    return host, n


def _params(C, K, seed):
    g = _gen(seed + 1)
    w = _f32(torch.randn(C, K, generator=g, dtype=F64) / math.sqrt(K))
    gamma = _f32(1.0 + 0.2 * torch.randn(C, generator=g, dtype=F64))
    beta = _f32(0.2 * torch.randn(C, generator=g, dtype=F64))
    acc = [_f32(torch.randn(*s, generator=g, dtype=F64)) for s in ((C, K), (C,), (C,))]
    return w, gamma, beta, acc


def _dy(shape, dtype, seed):
    return torch.randn(*shape, generator=_gen(seed + 2), dtype=F64).to(dtype)


def _dev(*ts):
    return [t.to("cuda", F64) for t in ts]


# ============================================================================================ GroupNorm mode
def run_gn(B, C, K, S, T0, *, dtype, act, kind="rand", seed=0):
    lib = _lib()
    host, n = _wave(B, T0, K, S, kind, seed)
    w, gamma, beta, (dw0, dg0, db0) = _params(C, K, seed)
    wave = Buf(host.numel(), F32, host)
    wb, gb, bb = Buf(C * K, F32, w), Buf(C, F32, gamma), Buf(C, F32, beta)
    nws = lib.st5_conv0_ws_floats(B, n, C, K, S)
    ws, y, mean, rstd = Buf(nws), Buf(B * T0 * C, dtype), Buf(B * C), Buf(B * C)
    rc = lib.st5_conv0_gn_gelu_fwd(P(wave.t), P(wb.t), P(gb.t), P(bb.t), P(y.t), DT[dtype], P(mean.t), P(rstd.t),
                                   P(ws.t), B, n, C, K, S, EPS, ACTS[act], ct.c_void_p(_st()))
    torch.cuda.synchronize()
    assert rc == 0, rc
    for buf, what in ((y, "y"), (mean, "mean"), (rstd, "rstd"), (ws, "ws")):
        buf.untouched(what)
    wave_d, w_d, g_d, b_d = _dev(host, w, gamma, beta)
    f = R.gn_forward(torch.nan_to_num(wave_d), w_d, g_d, b_d, S=S, eps=R.R.f32(EPS), act=act)
    bnd = R.gn_forward_bounds(f, R.R.unit(dtype))
    tag = f"gn_fwd {'bf16' if dtype == BF16 else 'f32'}"
    R.check(f"{tag} mean", mean.t.view(B, C), f["mean"], bnd["mean"], report=REPORT)
    R.check(f"{tag} rstd", rstd.t.view(B, C), f["rstd"], bnd["rstd"], report=REPORT)
    R.check(f"{tag} y", y.t.view(B, T0, C), f["y"], bnd["y"], report=REPORT)
    # the backward reads the reference statistics (as fp32), so that its statement does not depend on the forward's
    mean_in, rstd_in = _f32(f["mean"]), _f32(f["rstd"])
    del f, bnd
    dy = _dy((B, T0, C), dtype, seed)
    dyb = Buf(dy.numel(), dtype, dy)
    mb, rb = Buf(B * C, F32, mean_in), Buf(B * C, F32, rstd_in)
    dwb, dgb, dbb = Buf(C * K, F32, dw0), Buf(C, F32, dg0), Buf(C, F32, db0)
    ws = Buf(nws)
    rc = lib.st5_conv0_gn_gelu_bwd(P(dyb.t), P(wave.t), P(wb.t), P(gb.t), P(bb.t), P(mb.t), P(rb.t), P(dwb.t),
                                   P(dgb.t), P(dbb.t), P(ws.t), DT[dtype], B, n, C, K, S, ACTS[act], ct.c_void_p(_st()))
    torch.cuda.synchronize()
    assert rc == 0, rc
    for buf, what in ((dwb, "dw"), (dgb, "dgamma"), (dbb, "dbeta"), (ws, "ws")):
        buf.untouched(what)
    dw0_d, dg0_d, db0_d = _dev(dw0, dg0, db0)
    b = R.gn_backward(dy.to("cuda"), torch.nan_to_num(wave_d), w_d, g_d, b_d, *_dev(mean_in, rstd_in), S=S, act=act)
    bb_ = R.gn_backward_bounds(b, dw0_d, dg0_d, db0_d)
    tag = f"gn_bwd {'bf16' if dtype == BF16 else 'f32'}"
    R.check(f"{tag} dw", dwb.t.view(C, K), dw0_d + b["dw"], bb_["dw"], report=REPORT)
    R.check(f"{tag} dgamma", dgb.t, dg0_d + b["dgamma"], bb_["dgamma"], report=REPORT)
    R.check(f"{tag} dbeta", dbb.t, db0_d + b["dbeta"], bb_["dbeta"], report=REPORT)


def _cycle(i):
    return (F32, BF16)[i % 2], ("gelu", "gelu_tanh")[(i // 2) % 2]


@pytest.mark.parametrize("i,C", list(enumerate([1, 31, 33, 512, 800, 801, 1000, 1024])))
def test_gn_channels(i, C):
    """C > 512 runs as channel groups on grid.z; 801 and 1024 are the widths whose one-block backward could not launch."""
    dtype, act = _cycle(i)
    run_gn(2, C, 10, 5, 129, dtype=dtype, act=act, seed=i)


@pytest.mark.parametrize("i,K,S", [(i, K, S) for i, (K, S) in enumerate((K, S) for K in (1, 2, 10, 16)
                                                                         for S in (1, 5, 96))])
def test_gn_taps_and_strides(i, K, S):
    """S = 96: (127 S + K) floats is the largest staged segment under 48 KiB."""
    dtype, act = _cycle(i)
    run_gn(2, 33, K, S, 130, dtype=dtype, act=act, seed=10 + i)


@pytest.mark.parametrize("i,T0", list(enumerate([1, 127, 128, 129, 128 * 3 + 1])))
def test_gn_frames(i, T0):
    dtype, act = _cycle(i)
    run_gn(3, 64, 10, 5, T0, dtype=dtype, act=act, seed=20 + i)


@pytest.mark.parametrize("i,kind", list(enumerate(["const", "dc", "click", "silence"])))
def test_gn_waveforms(i, kind):
    """Zero variance (rstd = eps^-1/2), a DC offset of 100 under a 0.01 signal, a click on the pilot frame of every
    chunk, and silence."""
    for j, dtype in enumerate((F32, BF16)):
        run_gn(2, 96, 10, 5, 300, dtype=dtype, act=("gelu", "gelu_tanh")[(i + j) % 2], kind=kind, seed=30 + i)


@pytest.mark.parametrize("dtype", [BF16, F32])
def test_gn_bench_shape(dtype):
    """The ASR bench's layer 0: 8 utterances of 160 000 samples, K = 10, S = 5, C = 512."""
    run_gn(8, 512, 10, 5, (160000 - 10) // 5 + 1, dtype=dtype, act="gelu", seed=40)


# ============================================================================================ LayerNorm mode
def run_ln(B, C, K, S, T0, *, dtype, act, kind="rand", seed=0):
    lib = _lib()
    host, n = _wave(B, T0, K, S, kind, seed)
    w, gamma, beta, (dw0, dg0, db0) = _params(C, K, seed)
    wave = Buf(host.numel(), F32, host)
    wb, gb, bb = Buf(C * K, F32, w), Buf(C, F32, gamma), Buf(C, F32, beta)
    y, mean, rstd = Buf(B * T0 * C, dtype), Buf(B * T0), Buf(B * T0)
    rc = lib.st5_conv0_ln_gelu_fwd(P(wave.t), P(wb.t), P(gb.t), P(bb.t), P(y.t), DT[dtype], P(mean.t), P(rstd.t),
                                   B, n, C, K, S, EPS, ACTS[act], ct.c_void_p(_st()))
    torch.cuda.synchronize()
    assert rc == 0, rc
    for buf, what in ((y, "y"), (mean, "mean"), (rstd, "rstd")):
        buf.untouched(what)
    wave_d, w_d, g_d, b_d = _dev(host, w, gamma, beta)
    wave_d = torch.nan_to_num(wave_d)
    f = R.ln_forward(wave_d, w_d, g_d, b_d, S=S, eps=R.R.f32(EPS), act=act)
    bnd = R.ln_forward_bounds(f, R.R.unit(dtype))
    tag = f"ln_fwd {'bf16' if dtype == BF16 else 'f32'}"
    R.check(f"{tag} mean", mean.t, f["mean"].reshape(-1), bnd["mean"], report=REPORT)
    R.check(f"{tag} rstd", rstd.t, f["rstd"].reshape(-1), bnd["rstd"], report=REPORT)
    R.check(f"{tag} y", y.t.view(B, T0, C), f["y"], bnd["y"], report=REPORT)
    # the backward reads the reference statistics (as fp32), so that its statement does not depend on the forward's
    mean_in, rstd_in = _f32(f["mean"].reshape(-1)), _f32(f["rstd"].reshape(-1))
    del f, bnd
    dy = _dy((B, T0, C), dtype, seed)
    dyb = Buf(dy.numel(), dtype, dy)
    mb, rb = Buf(B * T0, F32, mean_in), Buf(B * T0, F32, rstd_in)
    dwb, dgb, dbb = Buf(C * K, F32, dw0), Buf(C, F32, dg0), Buf(C, F32, db0)
    ws = Buf(lib.st5_conv0_ln_ws_floats(B, n, C, K, S))
    rc = lib.st5_conv0_ln_gelu_bwd(P(dyb.t), P(wave.t), P(wb.t), P(gb.t), P(bb.t), P(mb.t), P(rb.t), P(dwb.t),
                                   P(dgb.t), P(dbb.t), P(ws.t), DT[dtype], B, n, C, K, S, ACTS[act], ct.c_void_p(_st()))
    torch.cuda.synchronize()
    assert rc == 0, rc
    for buf, what in ((dwb, "dw"), (dgb, "dgamma"), (dbb, "dbeta"), (ws, "ws")):
        buf.untouched(what)
    dw0_d, dg0_d, db0_d = _dev(dw0, dg0, db0)
    b = R.ln_backward(dy.to("cuda"), wave_d, w_d, g_d, b_d, *_dev(mean_in, rstd_in), S=S, act=act)
    bb_ = R.ln_backward_bounds(b, dw0_d, dg0_d, db0_d, _sms())
    tag = f"ln_bwd {'bf16' if dtype == BF16 else 'f32'}"
    R.check(f"{tag} dw", dwb.t.view(C, K), dw0_d + b["dw"], bb_["dw"], report=REPORT)
    R.check(f"{tag} dgamma", dgb.t, dg0_d + b["dgamma"], bb_["dgamma"], report=REPORT)
    R.check(f"{tag} dbeta", dbb.t, db0_d + b["dbeta"], bb_["dbeta"], report=REPORT)


@pytest.mark.parametrize("i,C", list(enumerate([2, 62, 64, 66, 258, 512])))
def test_ln_channels(i, C):
    dtype, act = _cycle(i)
    run_ln(2, C, 10, 5, 150, dtype=dtype, act=act, seed=50 + i)


@pytest.mark.parametrize("i,K", list(enumerate([1, 10, 11, 16])))
def test_ln_taps(i, K):
    """K <= 10 and K > 10 are the two backward instantiations (KH = 5 and 8 tap pairs per warp)."""
    for j, dtype in enumerate((F32, BF16)):
        run_ln(2, 66, K, 3, 90, dtype=dtype, act=("gelu", "gelu_tanh")[(i + j) % 2], seed=60 + i)


@pytest.mark.parametrize("i,B,T0", [(0, 1, 1), (1, 1, 3), (2, 3, 5000)])
def test_ln_frames(i, B, T0):
    """Fewer frames than one CTA's 4 warp pairs, and more than the persistent grid of 2 x SMs CTAs visits at once."""
    for j, dtype in enumerate((F32, BF16)):
        run_ln(B, 258, 10, 5, T0, dtype=dtype, act=("gelu", "gelu_tanh")[(i + j) % 2], seed=70 + i)


@pytest.mark.parametrize("kind", ["const", "dc", "silence"])
def test_ln_waveforms(kind):
    run_ln(2, 64, 10, 5, 40, dtype=F32, act="gelu", kind=kind, seed=80)


# ============================================================================================ conv0 rejections
def _conv0_call(lib, mode, bufs, dtype, B, n, C, K, S, act, fwd):
    wave, w, g, b, y, mean, rstd, ws, dy, dw, dg, db = (P(t.t) for t in bufs)
    st = ct.c_void_p(_st())
    if mode == "gn":
        if fwd:
            return lib.st5_conv0_gn_gelu_fwd(wave, w, g, b, y, DT[dtype], mean, rstd, ws, B, n, C, K, S, EPS, act, st)
        return lib.st5_conv0_gn_gelu_bwd(dy, wave, w, g, b, mean, rstd, dw, dg, db, ws, DT[dtype], B, n, C, K, S, act,
                                         st)
    if fwd:
        return lib.st5_conv0_ln_gelu_fwd(wave, w, g, b, y, DT[dtype], mean, rstd, B, n, C, K, S, EPS, act, st)
    return lib.st5_conv0_ln_gelu_bwd(dy, wave, w, g, b, mean, rstd, dw, dg, db, ws, DT[dtype], B, n, C, K, S, act, st)


@pytest.mark.parametrize("mode,B,n,C,K,S,act,want", [
    ("gn", 0, 200, 32, 10, 5, 2, -2), ("gn", 2, 200, 0, 10, 5, 2, -2), ("gn", 2, 200, 1025, 10, 5, 2, -2),
    ("gn", 2, 200, 32, 0, 5, 2, -2), ("gn", 2, 200, 32, 17, 5, 2, -2), ("gn", 2, 200, 32, 10, 0, 2, -2),
    ("gn", 2, 200, 32, 10, 5, 1, -3), ("gn", 2, 200, 32, 10, 5, 3, -3), ("gn", 2, 9, 32, 10, 5, 2, -4),
    ("gn", 2, 20000, 32, 10, 97, 2, -5),
    ("ln", 0, 200, 32, 10, 5, 2, -2), ("ln", 2, 200, 33, 10, 5, 2, -2), ("ln", 2, 200, 514, 10, 5, 2, -2),
    ("ln", 2, 200, 32, 17, 5, 2, -2), ("ln", 2, 200, 32, 10, 0, 2, -2), ("ln", 2, 200, 32, 10, 5, 0, -3),
    ("ln", 2, 9, 32, 10, 5, 4, -4)])
def test_conv0_rejections_leave_buffers_untouched(mode, B, n, C, K, S, act, want):
    lib = _lib()
    Bp, Cp, Kp = max(B, 1), max(C, 2), max(K, 1)
    T0p = max(R.frames(n, Kp, max(S, 1)), 1)
    g = _gen(5)
    bufs = [Buf(Bp * n, F32, torch.randn(Bp * n, generator=g)), Buf(Cp * Kp, F32, torch.randn(Cp * Kp, generator=g)),
            Buf(Cp, F32, torch.ones(Cp)), Buf(Cp, F32, torch.zeros(Cp)), Buf(Bp * T0p * Cp, BF16),
            Buf(Bp * T0p * Cp, F32, torch.zeros(Bp * T0p * Cp)), Buf(Bp * T0p * Cp, F32, torch.ones(Bp * T0p * Cp)),
            Buf(1 << 16), Buf(Bp * T0p * Cp, BF16, torch.ones(Bp * T0p * Cp)), Buf(Cp * Kp, F32, torch.ones(Cp * Kp)),
            Buf(Cp, F32, torch.ones(Cp)), Buf(Cp, F32, torch.ones(Cp))]
    snaps = [b.snapshot() for b in bufs]
    for fwd in (True, False):
        rc = _conv0_call(lib, mode, bufs, BF16, B, n, C, K, S, act, fwd)
        torch.cuda.synchronize()
        assert rc == want, (fwd, rc)
        assert all(b.same_as(s) for b, s in zip(bufs, snaps)), f"rc {rc} ({'fwd' if fwd else 'bwd'}) wrote a buffer"


# ============================================================================================ decode attention
class Decode:
    """q / k / v in fused q|k|v rows of width 3 H 64 + 8 (NaN in the blocks a call does not own), Tbuf >= Tk key rows
    per utterance (rows >= Tk NaN), masked keys' K / V rows NaN; out rows of pitch H 64 + 32 (gaps NaN)."""

    def __init__(self, q, k, v, key_pad, dtype, Tbuf=None, probs=True, ws=True):
        B, H, Tk, _ = k.shape
        self.B, self.H, self.Tk, self.dtype = B, H, Tk, dtype
        Tbuf = Tbuf or Tk + 3
        W = 3 * H * 64 + 8
        qh = torch.full((B, W), NAN, dtype=F32)
        qh[:, :H * 64] = q.reshape(B, H * 64).float()
        kv = torch.full((B, Tbuf, W), NAN, dtype=F32)
        kv[:, :Tk, H * 64:2 * H * 64] = k.transpose(1, 2).reshape(B, Tk, H * 64).float()
        kv[:, :Tk, 2 * H * 64:3 * H * 64] = v.transpose(1, 2).reshape(B, Tk, H * 64).float()
        if key_pad is not None:
            kv[:, :Tk][key_pad.bool()] = NAN
        self.qb, self.kvb = Buf(qh.numel(), dtype, qh), Buf(kv.numel(), dtype, kv)
        self.o_bs = H * 64 + 32
        self.out = Buf(B * self.o_bs, dtype)
        self.probs = Buf(B * H * Tk) if probs else None
        nws = _lib().st5_attn_decode_ws_floats(B, H, Tk, int(probs))
        self.ws = Buf(nws) if ws and nws > 0 else None
        self.kp = key_pad.cuda().contiguous() if key_pad is not None else None
        self.W, self.Tbuf = W, Tbuf

    def args(self, scale, k_off=0, v_off=0, ld_add=0, bs_add=0):
        H = self.H
        a = _lib_args()
        a.B, a.H, a.Tk, a.dtype = self.B, H, self.Tk, DT[self.dtype]
        esz = 4 if self.dtype == F32 else 2
        base = self.kvb.t.data_ptr()
        a.q, a.q_bs = self.qb.t.data_ptr(), self.W
        a.k, a.k_ld, a.k_bs = base + (H * 64 + k_off) * esz, self.W + ld_add, self.Tbuf * self.W + bs_add
        a.v, a.v_ld, a.v_bs = base + (2 * H * 64 + v_off) * esz, self.W, self.Tbuf * self.W
        a.key_pad = self.kp.data_ptr() if self.kp is not None else None
        a.out, a.o_bs = self.out.t.data_ptr(), self.o_bs
        a.probs = self.probs.t.data_ptr() if self.probs is not None else None
        a.scale = scale
        a.ws = self.ws.t.data_ptr() if self.ws is not None else None
        return a

    def run(self, scale, **kw):
        a = self.args(scale, **kw)
        rc = _lib().st5_attn_decode_fwd(ct.byref(a), ct.c_void_p(_st()))
        torch.cuda.synchronize()
        return rc

    def bufs(self):
        return [b for b in (self.qb, self.kvb, self.out, self.probs, self.ws) if b is not None]

    def out_rows(self):
        o = self.out.t.view(self.B, self.o_bs)
        assert bool(torch.isnan(o[:, self.H * 64:].float()).all()), "out: gap between rows written"
        return o[:, :self.H * 64].reshape(self.B, self.H, 64)


def _lib_args():
    from speecht5_b200 import _lib as L
    return L.AttnDecodeArgs()


def _decode_inputs(B, H, Tk, dtype, seed, std=3.0):
    q, k, v, _ = A.make_inputs(B, H, 1, Tk, std=std, seed=seed, dtype=dtype)
    return q[:, :, 0], k, v


def _check_decode(name, d, q, k, v, key_pad, scale):
    f = A.decode_forward(q, k, v, scale=A.np.float32(scale).item(), key_pad=key_pad)
    b = A.decode_bounds(f, u=R.R.unit(d.dtype))
    out = d.out_rows()
    for buf in d.bufs():
        buf.untouched(name)
    A.check(f"{name} out", out.cpu(), f["out"][:, :, 0], b["out"], dims="bhc", report=REPORT)
    if d.probs is not None:
        A.check(f"{name} probs", d.probs.t.view(d.B, d.H, d.Tk).cpu(), f["P"][:, :, 0], b["P"], dims="bhj",
                report=REPORT)
    return out.clone(), None if d.probs is None else d.probs.t.clone()


def _ragged(B, Tk, seed):
    """key_pad with utterance b holding its first L_b keys (L_0 = Tk), as the batched synthesis pads."""
    g = _gen(seed)
    L = [Tk] + [int(torch.randint(1, Tk + 1, (1,), generator=g)) for _ in range(B - 1)]
    return (torch.arange(Tk)[None, :] >= torch.tensor(L)[:, None]).to(torch.uint8)


@pytest.mark.parametrize("i,Tk", list(enumerate([1, 63, 64, 65, 128, 129, 1500, 4000])))
@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("probs", [True, False])
def test_decode(i, Tk, dtype, probs):
    B, H = [(1, 1), (3, 12), (32, 16)][i % 3]
    if Tk == 4000:
        B = 3
    q, k, v = _decode_inputs(B, H, Tk, dtype, seed=100 + i)
    key_pad = None if i % 2 == 0 else _ragged(B, Tk, i)
    d = Decode(q, k, v, key_pad, dtype, probs=probs)
    assert d.run(0.125) == 0
    _check_decode(f"decode {'bf16' if dtype == BF16 else 'f32'}", d, q, k, v, key_pad, 0.125)


@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("Tk", [40, 200])
def test_decode_edge_masks(dtype, Tk):
    """One utterance with a single key, one whose keys 64..127 are all masked (a dead split between valid ones), one
    with every key masked (zeros), one ragged; the result of each utterance does not depend on the buffer's key span."""
    B, H = 4, 12
    q, k, v = _decode_inputs(B, H, Tk, dtype, seed=7)
    kp = torch.zeros(B, Tk, dtype=torch.uint8)
    kp[0, 1:] = 1
    kp[1, 64:128] = 1
    kp[2, :] = 1
    kp[3, Tk // 2:] = 1
    d = Decode(q, k, v, kp, dtype)
    assert d.run(0.125) == 0
    out, pr = _check_decode(f"decode {'bf16' if dtype == BF16 else 'f32'}", d, q, k, v, kp, 0.125)
    assert bool((out[2] == 0).all()) and bool((pr.view(B, H, Tk)[2] == 0).all())
    # the same utterances inside a wider key span: bit-identical outputs and probabilities on their valid keys
    T2 = Tk + 150
    k2 = torch.cat([k, torch.randn(B, H, 150, 64).to(dtype)], 2)
    v2 = torch.cat([v, torch.randn(B, H, 150, 64).to(dtype)], 2)
    kp2 = torch.cat([kp, torch.ones(B, 150, dtype=torch.uint8)], 1)
    d2 = Decode(q, k2, v2, kp2, dtype)
    assert d2.run(0.125) == 0
    w = torch.int32 if dtype == F32 else torch.int16
    assert torch.equal(d2.out_rows().contiguous().view(w), out.contiguous().view(w))
    p2 = d2.probs.t.view(B, H, T2)
    assert torch.equal(p2[..., :Tk].contiguous().view(torch.int32), pr.view(B, H, Tk).contiguous().view(torch.int32))
    assert bool((p2[..., Tk:] == 0).all())


@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("Tk", [64, 129])
def test_decode_underflowing_scores(dtype, Tk):
    """Scores spread over thousands: exp(s - max) underflows to exactly 0 for most keys, and a whole split's maximum
    sits far below the global one."""
    B, H = 2, 4
    q, k, v = _decode_inputs(B, H, Tk, dtype, seed=9, std=3.0)
    d = Decode(q, k, v, None, dtype)
    scale = 64.0
    assert d.run(scale) == 0
    _, pr = _check_decode(f"decode {'bf16' if dtype == BF16 else 'f32'} large", d, q, k, v, None, scale)
    assert int((pr == 0).sum()) > 0


@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("what,want", [("ws", -5), ("k", -6), ("v", -6), ("ld", -6), ("bs", -6)])
def test_decode_rejections_leave_buffers_untouched(dtype, what, want):
    B, H, Tk = 2, 2, 100
    q, k, v = _decode_inputs(B, H, Tk, dtype, seed=11)
    d = Decode(q, k, v, _ragged(B, Tk, 3), dtype, ws=what != "ws")
    snaps = [b.snapshot() for b in d.bufs()]
    kw = dict(k=dict(k_off=1), v=dict(v_off=1), ld=dict(ld_add=1), bs=dict(bs_add=1)).get(what, {})
    assert d.run(0.125, **kw) == want
    assert all(b.same_as(s) for b, s in zip(d.bufs(), snaps))

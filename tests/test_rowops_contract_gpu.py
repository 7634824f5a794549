"""-m gpu: the LayerNorm, BatchNorm, posenc, colsum, cast, activation, lrelu_pad, dropout, sumsq and Adam entry points of
include/speecht5_b200.h called directly (speecht5_b200/kernels.py), against the fp64 statement of tests/rowops_ref.py
with ELEMENTWISE bounds, on buffers laid out here with NaN sentinels everywhere the contract does not let a kernel read
or write:
  - every output sits inside a NaN buffer with guard zones; strided operands (BatchNorm x / y / dy / dx, colsum x,
    cast src / dst) have NaN padding columns;
  - accumulated outputs (dgamma, dbeta, dxsum, demb, dalpha, colsum with accumulate, sumsq) start non-zero, scratch
    (the BatchNorm scratch) starts NaN;
  - shapes sit on every branch of the launchers: the persistent LayerNorm backward at one and two rows per warp (the SM
    count is read from the device), the fused vs two-kernel backward, the NCH = 3 / 4 instantiations, the vector and
    scalar BatchNorm / posenc / colsum / Adam kernels, colsum modes 0 / 1 / 2, and the scalar tails.
The largest err / bound of every entry point is printed at the end of the module (run with -s)."""
import math

import pytest
import torch

import rowops_ref as R

pytestmark = pytest.mark.gpu

NAN = float("nan")
G = 64  # guard elements before and after every buffer
SEED, OFFSET = 4321, 11
EPS = 1e-5
REPORT = {}
F32, BF16 = torch.float32, torch.bfloat16


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per entry point:")
        for k in sorted(REPORT):
            print(f"  {k:44s} {REPORT[k]:.3g}")


def _K():
    from speecht5_b200 import kernels as K
    return K


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Flat:
    """A contiguous [shape] tensor inside a NaN buffer with guard zones; `off` elements past the aligned start."""

    def __init__(self, shape, dtype, fill=None, off=0):
        n = math.prod(shape)
        self.flat = torch.full((2 * G + n + off,), NAN, dtype=dtype, device="cuda")
        self.lo, self.hi = G + off, G + off + n
        self.t = self.flat[self.lo:self.hi].view(shape)
        if fill is not None:
            self.t.copy_(fill.to(dtype) if torch.is_tensor(fill) else torch.full(shape, fill, dtype=dtype))

    def get(self):
        return self.t.cpu()

    def untouched(self, what):
        g = torch.cat([self.flat[:self.lo], self.flat[self.hi:]]).float()
        assert bool(torch.isnan(g).all()), f"{what}: guard zone written"


class Strided:
    """Logical [rows, cols] at row pitch ld > cols inside a NaN buffer: padding columns and guards stay NaN."""

    def __init__(self, rows, cols, ld, dtype, fill=None):
        self.rows, self.cols, self.ld = rows, cols, ld
        self.flat = torch.full((2 * G + rows * ld,), NAN, dtype=dtype, device="cuda")
        self.t = self.flat[G:G + rows * ld].view(rows, ld)[:, :cols]
        if fill is not None:
            self.t.copy_(fill.to(dtype))

    def get(self):
        return self.t.cpu()

    def untouched(self, what):
        inside = torch.zeros_like(self.flat, dtype=torch.bool)
        inside[G:G + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols] = True
        assert bool(torch.isnan(self.flat[~inside].float()).all()), f"{what}: written outside [rows, cols]"


def _rnd(shape, seed, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale + shift


def _u(dt):
    return R.unit(dt)


# ============================================================================================ LayerNorm
def _ln_cases():
    cases = []  # rows "16sm+k": 16 x the device's SM count + k (one vs. two rows per warp of the persistent backward)
    for C in (8, 80, 256, 760, 768, 776, 1024):
        for dt in ("f32", "bf16"):
            cases.append(dict(C=C, dt=dt, rows=65, res="same", drop=0.1))
    cases += [
        dict(C=768, dt="bf16", rows=1, res="none", drop=0.0),
        dict(C=768, dt="bf16", rows=3, res="f32", drop=0.1, nulls=("s_out",)),
        dict(C=768, dt="bf16", rows=63, res="same", drop=0.1),                       # two-kernel backward
        dict(C=768, dt="bf16", rows=63, res="same", drop=0.1, dxsum=True),          # dxsum forces the fused one
        dict(C=768, dt="f32", rows=64, res="f32", drop=0.0, dxsum=True, dxsum_off=1, nulls=("mean_rstd_fwd",)),
        dict(C=1024, dt="bf16", rows=64, res="same", drop=0.1, dxsum=True, nulls=("ds",)),
        dict(C=256, dt="f32", rows=65, res="same", drop=0.0, dxsum=True, nulls=("dx",)),
        dict(C=512, dt="bf16", rows=200, res="same", drop=0.0, nulls=("dgamma",), dxsum=True),
        dict(C=512, dt="f32", rows=200, res="none", drop=0.0, nulls=("dbeta",)),
        dict(C=776, dt="bf16", rows="16sm-1", res="same", drop=0.1, dxsum=True),
        dict(C=768, dt="bf16", rows="16sm+1", res="same", drop=0.1, dxsum=True),
        dict(C=1024, dt="f32", rows="16sm+1", res="f32", drop=0.0),
        dict(C=768, dt="bf16", rows="16sm", res="none", drop=0.0, offset=True, const=True),
        dict(C=1024, dt="bf16", rows=10007, res="f32", drop=0.1, dxsum=True),
        dict(C=80, dt="f32", rows=65, res="same", drop=0.0, offset=True, const=True),
    ]
    return cases


LN_CASES = _ln_cases()


def _id(c):
    return "-".join(f"{k}{v}" if not isinstance(v, tuple) else f"{k}{'+'.join(v)}" for k, v in c.items())


@pytest.mark.parametrize("case", LN_CASES, ids=[_id(c) for c in LN_CASES])
def test_layernorm(cuda, case):
    K = _K()
    C, res, drop = case["C"], case["res"], case["drop"]
    dt = F32 if case["dt"] == "f32" else BF16
    u = _u(dt)
    rows = case["rows"]
    if isinstance(rows, str):
        rows = 16 * _sms() + int(rows[4:] or 0)
    nulls = case.get("nulls", ())
    x = _rnd((rows, C), 1).to(dt)
    shift = 100.0 if case.get("offset") else 0.0
    r = _rnd((rows, C), 2, shift=shift)
    if case.get("const"):
        x[::3] = 0
        r[::3] = 0.7 + shift
    r = r.to(F32 if res == "f32" else dt)
    gamma = (1.0 + 0.2 * _rnd(C, 3)).float()
    beta = (0.2 * _rnd(C, 4)).float()
    kp = R.keep((rows, C), drop, SEED, OFFSET) if drop > 0 else None
    dsc = R.D.drop_scale(drop)
    f = R.ln_forward(x, gamma, beta, eps=EPS, residual=None if res == "none" else r, kp=kp, dscale=dsc)
    b = R.ln_forward_bounds(f, u)

    xb, gb, bb = Flat((rows, C), dt, x), Flat((C,), F32, gamma), Flat((C,), F32, beta)
    rb = Flat((rows, C), r.dtype, r) if res != "none" else None
    y, s_out = Flat((rows, C), dt), Flat((rows, C), dt) if "s_out" not in nulls else None
    no_stats = "mean_rstd_fwd" in nulls
    mean, rstd = (None, None) if no_stats else (Flat((rows,), F32), Flat((rows,), F32))
    y32 = Flat((rows, C), F32) if res == "f32" else None
    K.ln_fwd(xb.t, rb.t if res == "same" else None, gb.t, bb.t, y.t, s_out.t if s_out else None,
             mean.t if mean else None, rstd.t if rstd else None, EPS, drop, SEED, OFFSET,
             residual_f32=rb.t if res == "f32" else None, y_f32=y32.t if y32 else None)
    torch.cuda.synchronize()
    n = f"ln_fwd[{case['dt']}]" if res != "f32" else f"ln_fwd_stream[{case['dt']}]"
    R.check(f"{n} y", y.get(), f["y"], b["y"], REPORT)
    y.untouched(n)
    if s_out is not None:
        R.check(f"{n} s", s_out.get(), f["s"], b["s"], REPORT)
        s_out.untouched(n)
    if mean is not None:
        R.check(f"{n} mean", mean.get(), f["mean"], b["mean"], REPORT)
        R.check(f"{n} rstd", rstd.get(), f["rstd"], b["rstd"], REPORT)
        mean.untouched(n)
        rstd.untouched(n)
    if y32 is not None:
        R.check(f"{n} y_f32", y32.get(), f["y"], b["y_f32"], REPORT)
        y32.untouched(n)

    # ---- backward from s as stored and the fp32 statistics of that s
    s_in = f["s"].to(dt)
    fs = R.ln_forward(s_in, gamma, beta, eps=EPS)
    m_in, r_in = fs["mean"].float(), fs["rstd"].float()
    dy = _rnd((rows, C), 5).to(dt)
    dx_null = "dx" in nulls
    bw = R.ln_backward(dy, s_in, m_in, r_in, gamma, kp=kp, dscale=dsc, dx_null=dx_null)
    bwb = R.ln_backward_bounds(bw, u, dx_null=dx_null)
    dyb, sb, mb, rsb = Flat((rows, C), dt, dy), Flat((rows, C), dt, s_in), Flat((rows,), F32, m_in), \
        Flat((rows,), F32, r_in)
    ds = Flat((rows, C), dt) if "ds" not in nulls else None
    dx = Flat((rows, C), dt) if not dx_null else None
    g0, b0 = _rnd(C, 6).float(), _rnd(C, 7).float()
    dgamma = Flat((C,), F32, g0) if "dgamma" not in nulls else None
    dbeta = Flat((C,), F32, b0) if "dbeta" not in nulls else None
    xs0 = _rnd(C, 8).float()
    dxsum = Flat((C,), F32, xs0, off=case.get("dxsum_off", 0)) if case.get("dxsum") else None
    K.ln_bwd(dyb.t, sb.t, mb.t, rsb.t, gb.t, ds.t if ds else None, dx.t if dx else None,
             dgamma.t if dgamma else None, dbeta.t if dbeta else None, drop, SEED, OFFSET,
             dxsum=dxsum.t if dxsum else None)
    torch.cuda.synchronize()
    n = f"ln_bwd[{case['dt']}]"
    if ds is not None:
        R.check(f"{n} ds", ds.get(), bw["ds"], bwb["ds"], REPORT)
        ds.untouched(n)
    if dx is not None:
        R.check(f"{n} dx", dx.get(), bw["dx"], bwb["dx"], REPORT)
        dx.untouched(n)
    for buf, init, key in ((dgamma, g0, "dgamma"), (dbeta, b0, "dbeta"), (dxsum, xs0, "dxsum")):
        if buf is not None:
            want = init.double() + bw[key]
            R.check(f"{n} {key} (+=)", buf.get(), want, bwb[key] + R.U32 * (want.abs() + init.double().abs()),
                    REPORT)
            buf.untouched(f"{n} {key}")


# ============================================================================================ BatchNorm
BN_CASES = [
    # (C, x_ld, y_ld, rows, dtype): ld % 8 == 0 with C % 8 == 0 selects the vector kernels
    (37, 41, 45, 255, "f32"), (37, 40, 48, 1, "bf16"), (37, 48, 40, 2, "f32"),
    (80, 88, 96, 256, "bf16"), (80, 84, 88, 257, "f32"), (80, 88, 96, 257, "f32"),
    (256, 264, 272, 255, "bf16"), (520, 528, 536, 256, "f32"), (520, 524, 528, 2, "bf16"),
    (80, 88, 96, 128 * 256 + 1, "bf16"), (37, 41, 45, 128 * 256 + 1, "f32"),
]


@pytest.mark.parametrize("act", ["none", "relu", "tanh"])
@pytest.mark.parametrize("C,x_ld,y_ld,rows,dts", BN_CASES)
def test_batchnorm(cuda, C, x_ld, y_ld, rows, dts, act):
    K = _K()
    dt = F32 if dts == "f32" else BF16
    u = _u(dt)
    x = _rnd((rows, C), 11, scale=1.5, shift=0.3).to(dt)
    gamma = (1.0 + 0.3 * _rnd(C, 12)).float()
    beta = (0.3 * _rnd(C, 13)).float()
    rm0, rv0 = _rnd(C, 14).float(), (0.5 + _rnd(C, 15).abs()).float()
    drop = 0.1 if rows % 2 else 0.0
    kp = R.keep((rows, C), drop, SEED, OFFSET) if drop > 0 else None
    dsc = R.D.drop_scale(drop)
    with_pre = act != "none" or rows == 255
    for training in (1, 0):
        f = R.bn_forward(x, gamma, beta, rm0, rv0, training=bool(training), momentum=0.1, eps=EPS, act_name=act,
                         kp=kp, dscale=dsc)
        b = R.bn_forward_bounds(f, u)
        xb = Strided(rows, C, x_ld, dt, x)
        yb = Strided(rows, C, y_ld, dt)
        ypre = Flat((rows, C), dt) if with_pre else None
        gb, bb = Flat((C,), F32, gamma), Flat((C,), F32, beta)
        rm, rv = Flat((C,), F32, rm0), Flat((C,), F32, rv0)
        sm, sr = Flat((C,), F32), Flat((C,), F32)
        scratch = Flat((2 * C,), F32)
        K.bn_fwd(xb.t, x_ld, gb.t, bb.t, rm.t, rv.t, sm.t, sr.t, yb.t, y_ld, ypre.t if ypre else None, rows, C,
                 training, 0.1, EPS, act, drop, SEED, OFFSET, scratch.t)
        torch.cuda.synchronize()
        n = f"bn_fwd[{dts}]" + ("" if training else " eval")
        R.check(f"{n} save_mean", sm.get(), f["mean"], b["save_mean"], REPORT)
        R.check(f"{n} save_rstd", sr.get(), f["rstd"], b["save_rstd"], REPORT)
        R.check(f"{n} y", yb.get(), f["y"], b["y"], REPORT)
        yb.untouched(n)
        if ypre is not None:
            R.check(f"{n} y_pre", ypre.get(), f["pre"], b["y_pre"], REPORT)
            ypre.untouched(n)
        if training:
            R.check(f"{n} running_mean", rm.get(), f["running_mean"], b["running_mean"], REPORT)
            R.check(f"{n} running_var", rv.get(), f["running_var"], b["running_var"], REPORT)
        else:
            assert torch.equal(rm.get(), rm0) and torch.equal(rv.get(), rv0), f"{n}: running statistics written"
        for t in (sm, sr, rm, rv, scratch):
            t.untouched(n)

    # ---- backward (training statistics), y_pre as stored
    f = R.bn_forward(x, gamma, beta, rm0, rv0, training=True, momentum=0.1, eps=EPS, act_name=act)
    m_in, r_in = f["mean"].float(), f["rstd"].float()
    pre_in = f["pre"].to(dt)
    dy = _rnd((rows, C), 16).to(dt)
    bw = R.bn_backward(dy, x, pre_in if with_pre else None, gamma, m_in, r_in, act_name=act, kp=kp, dscale=dsc)
    bwb = R.bn_backward_bounds(bw, u)
    d_ld = x_ld + 8
    dyb, xb = Strided(rows, C, y_ld, dt, dy), Strided(rows, C, x_ld, dt, x)
    ypre = Flat((rows, C), dt, pre_in) if with_pre else None
    dxb = Strided(rows, C, d_ld, dt)
    g0, b0 = _rnd(C, 17).float(), _rnd(C, 18).float()
    dg, db = Flat((C,), F32, g0), Flat((C,), F32, b0)
    scratch = Flat((2 * C,), F32)
    K.bn_bwd(dyb.t, y_ld, xb.t, x_ld, ypre.t if ypre else None, Flat((C,), F32, gamma).t, Flat((C,), F32, m_in).t,
             Flat((C,), F32, r_in).t, dxb.t, d_ld, dg.t, db.t, rows, C, act, drop, SEED, OFFSET, scratch.t)
    torch.cuda.synchronize()
    n = f"bn_bwd[{dts}]"
    R.check(f"{n} dx", dxb.get(), bw["dx"], bwb["dx"], REPORT)
    dxb.untouched(n)
    for buf, init, key in ((dg, g0, "dgamma"), (db, b0, "dbeta")):
        want = init.double() + bw[key]
        R.check(f"{n} {key} (+=)", buf.get(), want, bwb[key] + R.U32 * (want.abs() + init.double().abs()), REPORT)
        buf.untouched(n)
    scratch.untouched(n)


# ============================================================================================ posenc
@pytest.mark.parametrize("dts", ["f32", "bf16"])
@pytest.mark.parametrize("C,misalign,demb_off", [(37, 0, 0), (64, 0, 0), (64, 0, 1), (64, 1, 1), (768, 0, 0),
                                                 (768, 0, 1)])
@pytest.mark.parametrize("use_tokens", [True, False])
def test_posenc(cuda, C, misalign, demb_off, use_tokens, dts):
    K = _K()
    dt = F32 if dts == "f32" else BF16
    u = _u(dt)
    B, T, V, pad = 3, 45, 50, 1
    gen = torch.Generator().manual_seed(C)
    tokens = torch.randint(0, V, (B, T), generator=gen)
    tokens[0, :9] = 7
    tokens[2, -10:] = pad
    emb = _rnd((V, C), 21).float()
    pe = _rnd((T + 3, C), 22).float()
    x = _rnd((B, T, C), 23).to(dt)
    alpha = 1.3
    drop = 0.1 if C != 64 else 0.0
    kp = R.keep((B, T, C), drop, SEED, OFFSET) if drop > 0 else None
    dsc = R.D.drop_scale(drop)
    off = misalign * (4 // (2 if dt == BF16 else 4))  # 4 bytes: the scalar kernels
    tok_dev = tokens.cuda() if use_tokens else None
    embb, peb = Flat((V, C), F32, emb), Flat((T + 3, C), F32, pe)
    xb = Flat((B, T, C), dt, x, off=off)
    al = torch.tensor([alpha], dtype=F32, device="cuda")
    y = Flat((B, T, C), dt, off=off)
    K.posenc_fwd(tok_dev, embb.t if use_tokens else None, None if use_tokens else xb.t, peb.t, al, y.t, drop, SEED,
                 OFFSET)
    torch.cuda.synchronize()
    ref, bnd = R.posenc_forward(pe, R.f32(alpha), T, tokens=tokens if use_tokens else None, emb=emb,
                                x=None if use_tokens else x, kp=kp, dscale=dsc, u=u)
    n = f"posenc_fwd[{dts}]"
    R.check(f"{n} y", y.get(), ref, bnd, REPORT)
    y.untouched(n)

    dy = _rnd((B, T, C), 24).to(dt)
    bw = R.posenc_backward(dy, pe, T, tokens=tokens if use_tokens else None, padding_idx=pad, n_emb=V, kp=kp,
                           dscale=dsc)
    dyb = Flat((B, T, C), dt, dy, off=off)
    dx = Flat((B, T, C), dt, off=off) if C != 768 else None  # dx may be NULL
    e0 = _rnd((V, C), 25).float()
    demb = Flat((V, C), F32, e0, off=demb_off)
    a0 = torch.tensor([0.75], dtype=F32)
    dal = Flat((1,), F32, a0)
    K.posenc_bwd(dyb.t, tok_dev, pad, peb.t, dx.t if dx else None, demb.t if use_tokens else None, dal.t, drop, SEED,
                 OFFSET)
    torch.cuda.synchronize()
    n = f"posenc_bwd[{dts}]"
    if dx is not None:
        R.check(f"{n} dx", dx.get(), bw["dx"], bw["b_dx"] + u * bw["dx"].abs(), REPORT)
        dx.untouched(n)
    want = 0.75 + bw["dalpha"]
    R.check(f"{n} dalpha (+=)", dal.get()[0], want, bw["b_dalpha"] + R.U32 * (abs(float(want)) + 0.75), REPORT)
    dal.untouched(n)
    if use_tokens:
        want = e0.double() + bw["demb"]
        R.check(f"{n} demb (+=)", demb.get(), want, bw["b_demb"] + R.U32 * (want.abs() + e0.double().abs()), REPORT)
    else:
        assert torch.equal(demb.get(), e0), f"{n}: demb written without tokens"
    demb.untouched(n)


# ============================================================================================ colsum
COLSUM_CASES = [
    # rows, cols, ld, group_rows, dtype: vec_ok = cols, ld multiples of 4 (fp32) / 8 (bf16)
    (1000, 96, 104, 300, "f32"),   # mode 0, several row splits, ragged last group
    (173, 96, 104, 50, "f32"),     # mode 1 / 2: one split per group
    (173, 96, 104, 50, "bf16"),
    (2000, 512, 520, 0, "bf16"),   # one group
    (999, 37, 41, 250, "f32"),     # scalar kernel
    (999, 37, 41, 64, "bf16"),
    (64, 100, 102, 64, "f32"),     # ld not a multiple of 4: scalar
]


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("rows,cols,ld,gr,dts", COLSUM_CASES)
def test_colsum(cuda, rows, cols, ld, gr, dts, accumulate):
    K = _K()
    dt = F32 if dts == "f32" else BF16
    x = _rnd((rows, cols), 31).to(dt)
    ref, bnd = R.colsum(x, gr)
    groups = ref.shape[0]
    xb = Strided(rows, cols, ld, dt, x)
    o0 = _rnd((groups, cols), 32).float()
    out = Flat((groups, cols), F32, o0 if accumulate else None)
    K.colsum(xb.t, out.t, group_rows=gr, accumulate=accumulate, ld=ld)
    torch.cuda.synchronize()
    want = ref + (o0.double() if accumulate else 0.0)
    R.check(f"colsum[{dts}]", out.get(), want, bnd + R.U32 * want.abs() + (R.U32 * o0.double().abs() if accumulate
                                                                          else 0.0), REPORT)
    out.untouched("colsum")


# ============================================================================================ elementwise
ALL_BF16 = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(BF16)  # every bf16 bit pattern
ACTS = ["none", "relu", "gelu", "tanh", "gelu_tanh"]


def _nonfinite_fwd(x, act):
    """The kernels' value at a non-finite input (stated in the header next to the ST5_ACT_* ids)."""
    x = x.double()
    out = torch.full_like(x, NAN)
    pinf, ninf = x == math.inf, x == -math.inf
    if act == "none":
        out = x.clone()
    elif act == "relu":  # fmaxf: NaN -> 0
        out = torch.where(torch.isnan(x), torch.zeros_like(x), x.clamp_min(0))
    elif act == "tanh":
        out[pinf], out[ninf] = 1.0, -1.0
    else:  # gelu forms: +inf -> +inf, -inf -> NaN (-inf * 0), NaN -> NaN
        out[pinf] = math.inf
    return out


def _same(got, want):
    got, want = got.double(), want.double()
    return bool(((got == want) | (torch.isnan(got) & torch.isnan(want))).all())


def _sweep_f32():
    dense = torch.linspace(-10, 10, 200001, dtype=F32)
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (200000,), generator=torch.Generator().manual_seed(5),
                         dtype=torch.int64).to(torch.int32).view(F32)
    return torch.cat([dense, bits, torch.tensor([0.0, -0.0, math.inf, -math.inf, NAN, 3.0e38, -3.0e38])])


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("dts", ["bf16", "f32"])
def test_act_fwd_every_input(cuda, act, dts):
    K = _K()
    dt = F32 if dts == "f32" else BF16
    x = ALL_BF16.clone() if dt == BF16 else _sweep_f32()
    n = x.numel()
    xb, y = Flat((n,), dt, x), Flat((n,), dt)
    K.act_fwd(xb.t, y.t, act)
    torch.cuda.synchronize()
    got = y.get()
    y.untouched(f"act_fwd[{dts},{act}]")
    fin = torch.isfinite(x)
    R.check(f"act_fwd[{dts},{act}]", got[fin], R.act(x[fin], act), R.act_fwd_bound(x[fin], act, _u(dt)), REPORT)
    assert _same(got[~fin], _nonfinite_fwd(x[~fin], act)), f"act_fwd[{dts},{act}]: non-finite inputs"
    if act in ("none", "relu"):  # exact
        want = x.double().clamp_min(0) if act == "relu" else x.double()
        assert bool((got.double()[fin] == want[fin]).all())


def test_gelu_tanh_error_over_all_bf16_inputs(cuda):
    """ST5_ACT_GELU_TANH evaluated in fp32 (st5_act_fwd, fp32 storage) on every finite bf16 value, against the erf
    GELU: the figure the header states."""
    K = _K()
    x = ALL_BF16.float()
    x = x[torch.isfinite(x)]
    xb, y = Flat((x.numel(),), F32, x), Flat((x.numel(),), F32)
    K.act_fwd(xb.t, y.t, "gelu_tanh")
    torch.cuda.synchronize()
    ref = R.gelu(x)
    err = (y.get().double() - ref).abs()
    i = int(err.argmax())
    print(f"\nGELU_TANH vs erf GELU over all finite bf16 inputs: max |err| {float(err[i]):.3g} at x = {float(x[i]):.4g}")
    REPORT["gelu_tanh |err| (abs)"] = float(err[i])
    R.check("act_fwd[f32,gelu_tanh] all bf16", y.get(), ref, R.GELU_TANH_ABS + R.GELU_TANH_REL * ref.abs()
            + R.C_EW * R.U32 * ref.abs(), REPORT)
    # csrc/kernels.cuh: below half a bf16 ulp of the output wherever |y| > 0.13
    big = ref.abs() > 0.13
    half_ulp = torch.ldexp(torch.ones_like(ref), torch.frexp(ref)[1] - 9)
    assert bool((err[big] < half_ulp[big]).all()), "GELU_TANH: error of half a bf16 ulp or more at |y| > 0.13"


@pytest.mark.parametrize("act", ["relu", "gelu", "tanh", "gelu_tanh", "none"])
@pytest.mark.parametrize("dts", ["bf16", "f32"])
def test_act_bwd_every_input(cuda, act, dts):
    K = _K()
    dt = F32 if dts == "f32" else BF16
    pre = ALL_BF16.clone() if dt == BF16 else _sweep_f32()
    n = pre.numel()
    drop = 0.1
    dy = _rnd(n, 41).to(dt)
    kp = R.keep((n,), drop, SEED, OFFSET)
    g = dy.double() * kp * R.D.drop_scale(drop)
    dyb, preb, out = Flat((n,), dt, dy), Flat((n,), dt, pre), Flat((n,), dt)
    K.act_bwd(dyb.t, preb.t, out.t, act, drop, SEED, OFFSET)
    torch.cuda.synchronize()
    got = out.get()
    out.untouched("act_bwd")
    p64 = pre.double()
    fin = torch.isfinite(p64)
    if act == "gelu_tanh":  # x * x overflows fp32 from 2^64 on: the derivative evaluates to NaN there
        fin &= p64.abs() < 2.0 ** 64
    ref, bnd = R.act_bwd_bound(g[fin], pre[fin], act, _u(dt))
    R.check(f"act_bwd[{dts},{act}]", got[fin], ref, bnd, REPORT)
    # non-finite pre: relu -> 0 for NaN / -inf and g for +inf; tanh -> 0 (1 - 1) for +-inf; none -> g; gelu forms NaN
    gn = g[~fin]
    pn = p64[~fin]
    if act == "relu":
        want = torch.where(pn == math.inf, gn, torch.zeros_like(gn))
    elif act == "tanh":
        want = torch.where(torch.isnan(pn), torch.full_like(gn, NAN), gn * 0.0)
    elif act == "none":
        want = gn
    else:
        want = torch.full_like(gn, NAN)
    assert _same(got[~fin].double(), want.to(dt).double()), f"act_bwd[{dts},{act}]: non-finite inputs"


@pytest.mark.parametrize("n", [1, 7, 8, 9, 4097])
@pytest.mark.parametrize("dts", ["bf16", "f32"])
def test_act_fwd_tails(cuda, n, dts):
    K = _K()
    dt = F32 if dts == "f32" else BF16
    x = _rnd(n, n).to(dt)
    xb, y = Flat((n,), dt, x), Flat((n,), dt)
    K.act_fwd(xb.t, y.t, "gelu")
    torch.cuda.synchronize()
    R.check(f"act_fwd[{dts},gelu] tails", y.get(), R.act(x, "gelu"), R.act_fwd_bound(x, "gelu", _u(dt)), REPORT)
    y.untouched("act_fwd tails")


@pytest.mark.parametrize("slope", [0.1, 1.0])
def test_lrelu_pad_every_input(cuda, slope):
    K = _K()
    x = ALL_BF16.view(2, 4096, 8)
    for d, ph, pad, n_in in ((1, 0, 3, 4102), (2, 1, 5, 2050), (3, 2, 0, 1365)):
        xb = Flat((2, 4096, 8), BF16, x)
        out = Flat((2, n_in, 8), BF16)
        K.lrelu_pad(xb.t, out.t, d, ph, pad, slope)
        torch.cuda.synchronize()
        got = out.get()
        out.untouched("lrelu_pad")
        # exactly one rounding: bf16(fp32(x * slope)) on x <= 0, x itself otherwise; zeros outside [0, T)
        x32 = x.float()
        lr = torch.where(x32 > 0, x32, x32 * R.f32(slope)).to(BF16)
        want = torch.zeros(2, n_in, 8, dtype=BF16)
        src = ph + d * torch.arange(n_in) - pad
        ok = (src >= 0) & (src < 4096)
        want[:, ok] = lr[:, src[ok]]
        same = (got.view(torch.int16) == want.view(torch.int16)) | (torch.isnan(got.float()) & torch.isnan(want.float()))
        assert bool(same.all()), f"lrelu_pad d={d} ph={ph}: {int((~same).sum())} elements differ"


def test_cast_bf16_hi_lo(cuda):
    K = _K()
    v = _sweep_f32()
    v = v[: (v.numel() // 97) * 97].view(-1, 97)
    rows, cols = v.shape
    src = Strided(rows, cols, 101, F32, v)
    hi, lo = Strided(rows, cols, 104, BF16), Strided(rows, cols, 104, BF16)
    K.cast_bf16(src.t, hi.t, lo.t)
    torch.cuda.synchronize()
    want_hi = v.to(BF16)
    want_lo = (v - want_hi.float()).to(BF16)
    for got, want, w in ((hi.get(), want_hi, "hi"), (lo.get(), want_lo, "lo")):
        same = (got.view(torch.int16) == want.view(torch.int16)) | (torch.isnan(got.float()) & torch.isnan(want.float()))
        assert bool(same.all()), f"cast_bf16 {w}: {int((~same).sum())} elements differ from round-to-nearest-even"
    hi.untouched("cast hi")
    lo.untouched("cast lo")


def test_dropout_p0_is_a_copy(cuda):
    K = _K()
    for dt in (F32, BF16):
        x = _rnd(1001, 3).to(dt)
        xb, y = Flat((1001,), dt, x), Flat((1001,), dt)
        K.dropout(xb.t, y.t, 0.0, SEED, OFFSET)
        torch.cuda.synchronize()
        assert torch.equal(y.get().view(torch.int16 if dt == BF16 else torch.int32),
                           x.view(torch.int16 if dt == BF16 else torch.int32))
        y.untouched("dropout p=0")


@pytest.mark.parametrize("n", [1, 3, 4, 5, 100003, 2 ** 25 + 3])
def test_sumsq(cuda, n):
    K = _K()
    x = (torch.randn(n, generator=torch.Generator().manual_seed(n)) * 0.01).float()
    xb = Flat((n,), F32, x)
    out = Flat((1,), F32, torch.tensor([0.5]))
    K.sumsq(xb.t, out.t)
    torch.cuda.synchronize()
    s, b = R.sumsq(x)
    R.check("sumsq (+=)", out.get()[0], 0.5 + s, b + R.U32 * (0.5 + s), REPORT)
    out.untouched("sumsq")


# ============================================================================================ Adam
ADAM_HP = dict(lr=0.05, beta1=0.9, beta2=0.98, eps=1e-6)


def _adam_run(n, off, shadow_off, *, wd, max_norm, gmul, step, lr_dev, step_dev, gn2=None, with_shadow=True,
              seed=0, state=None):
    """One st5_adam_step on slices at float offset `off` (shadow at bf16 offset shadow_off); returns (before, after
    tensors on the host, grad, gn2)."""
    K = _K()
    gen = torch.Generator().manual_seed(seed)
    if state is None:
        p = torch.randn(n, generator=gen)
        m = 0.1 * torch.randn(n, generator=gen)
        v = 0.01 * torch.rand(n, generator=gen)
    else:
        p, m, v = state
    g = torch.randn(n, generator=gen)
    if gn2 is None:
        gn2 = float((g.double() ** 2).sum())
    bufs = [Flat((n,), F32, t, off=off) for t in (p, g, m, v)]
    sh = Flat((n,), BF16, off=shadow_off) if with_shadow else None
    gn = torch.tensor([gn2], dtype=F32, device="cuda")
    lr_t = torch.tensor([ADAM_HP["lr"]], dtype=F32, device="cuda") if lr_dev else None
    st_t = torch.tensor([step], dtype=torch.int64, device="cuda") if step_dev else None
    host_step = 1 if step_dev else step
    host_lr = 123.0 if lr_dev else ADAM_HP["lr"]  # ignored when lr_dev is given
    K.adam_step(bufs[0].t, bufs[1].t, bufs[2].t, bufs[3].t, sh.t if sh else None, host_lr, ADAM_HP["beta1"],
                ADAM_HP["beta2"], ADAM_HP["eps"], wd, host_step, gn, max_norm, gmul, lr_dev=lr_t, step_dev=st_t)
    torch.cuda.synchronize()
    for b in bufs:
        b.untouched("adam_step")
    if sh is not None:
        sh.untouched("adam_step shadow")
    return (p, m, v), [b.get() for b in bufs], (sh.get() if sh else None), g, gn2


ADAM_CASES = [
    # n, float offset, shadow offset (bf16 elements), wd, max_norm, grad_mul, lr_dev, step_dev
    (4096, 0, 0, 0.0, 0.0, 1.0, False, False),
    (4097, 0, 0, 0.1, 1.0, 0.5, True, True),     # the trainer's combination (host step = 1)
    (4098, 1, 0, 0.1, 1e4, 0.5, True, False),
    (4099, 2, 4, 0.0, 1.0, 0.25, False, True),   # shadow 8-byte but not 16-byte aligned
    (4099, 0, 4, 0.1, 5.0, 1.0, False, False),
    (7, 0, 1, 0.1, 1.0, 0.5, True, True),        # 2-byte shadow offset: scalar path
    (1, 3, 0, 0.0, 0.0, 1.0, False, False),
]


@pytest.mark.parametrize("with_shadow", [True, False])
@pytest.mark.parametrize("n,off,soff,wd,max_norm,gmul,lr_dev,step_dev", ADAM_CASES)
def test_adam_step(cuda, n, off, soff, wd, max_norm, gmul, lr_dev, step_dev, with_shadow):
    step = 3
    before, after, sh, g, gn2 = _adam_run(n, off, soff, wd=wd, max_norm=max_norm, gmul=gmul, step=step, lr_dev=lr_dev,
                                          step_dev=step_dev, with_shadow=with_shadow, seed=n)
    p, m, v = before
    ref = R.adam_step(p, g, m, v, **ADAM_HP, weight_decay=wd, step=step, grad_norm_sq=gn2, max_norm=max_norm,
                      grad_mul=gmul)
    bnd = R.adam_bounds(before, ref, **ADAM_HP, weight_decay=wd, step=step, device_step=step_dev)
    n_ = "adam_step"
    R.check(f"{n_} p", after[0], ref["p"], bnd["p"], REPORT)
    R.check(f"{n_} m", after[2], ref["m"], bnd["m"], REPORT)
    R.check(f"{n_} v", after[3], ref["v"], bnd["v"], REPORT)
    assert torch.equal(after[1], g), "adam_step: gradient written"
    if sh is not None:  # the shadow is exactly RNE of the kernel's own p
        assert torch.equal(sh.view(torch.int16), after[0].to(BF16).view(torch.int16)), "adam_step: shadow != bf16(p)"


@pytest.mark.parametrize("gn2", [NAN, math.inf])
def test_adam_step_non_finite_norm_is_a_no_op(cuda, gn2):
    K = _K()
    n = 1027
    p, g, m, v = (torch.randn(n, generator=torch.Generator().manual_seed(i)) for i in range(4))
    v = v.abs()
    bufs = [Flat((n,), F32, t) for t in (p, g, m, v)]
    sh0 = p.to(BF16)
    sh = Flat((n,), BF16, sh0)
    gn = torch.tensor([gn2], dtype=F32, device="cuda")
    K.adam_step(bufs[0].t, bufs[1].t, bufs[2].t, bufs[3].t, sh.t, 1e-3, 0.9, 0.98, 1e-6, 0.1, 1, gn, 1.0, 1.0,
                lr_dev=torch.tensor([1e-3], device="cuda"), step_dev=torch.tensor([4], device="cuda"))
    torch.cuda.synchronize()
    for b, t in zip(bufs, (p, g, m, v)):
        assert torch.equal(b.get().view(torch.int32), t.view(torch.int32)), "adam_step changed state on a non-finite norm"
    assert torch.equal(sh.get().view(torch.int16), sh0.view(torch.int16))


def test_adam_twenty_step_trajectory(cuda):
    """20 updates of the trainer's form (lr_dev, step_dev, clip, weight decay), each against fp64 from the state the
    kernel left, and the final parameters against a pure fp64 trajectory."""
    n = 1025
    gen = torch.Generator().manual_seed(77)
    state = (torch.randn(n, generator=gen), torch.zeros(n), torch.zeros(n))
    p64, m64, v64 = (t.double() for t in state)
    for step in range(1, 21):
        before, after, sh, g, gn2 = _adam_run(n, 0, 0, wd=0.01, max_norm=1.0, gmul=0.5, step=step, lr_dev=True,
                                              step_dev=True, seed=1000 + step, state=state)
        ref = R.adam_step(before[0], g, before[1], before[2], **ADAM_HP, weight_decay=0.01, step=step,
                          grad_norm_sq=gn2, max_norm=1.0, grad_mul=0.5)
        bnd = R.adam_bounds(before, ref, **ADAM_HP, weight_decay=0.01, step=step, device_step=True)
        R.check("adam_step p (20 steps)", after[0], ref["p"], bnd["p"], REPORT)
        R.check("adam_step m (20 steps)", after[2], ref["m"], bnd["m"], REPORT)
        R.check("adam_step v (20 steps)", after[3], ref["v"], bnd["v"], REPORT)
        state = (after[0], after[2], after[3])
        full = R.adam_step(p64, g, m64, v64, **ADAM_HP, weight_decay=0.01, step=step, grad_norm_sq=gn2, max_norm=1.0,
                           grad_mul=0.5)
        p64, m64, v64 = full["p"], full["m"], full["v"]
    # fp32 state drift over 20 updates stays at the fp32 level of the parameters
    assert float((state[0].double() - p64).abs().max()) <= 20 * 16 * R.U32 * float(p64.abs().max())


# ============================================================================================ rejected configurations
def _raises(fn, match):
    with pytest.raises(RuntimeError, match=match):
        fn()


def test_rejected_configurations_leave_buffers_untouched(cuda):
    K = _K()

    def nan_all(*bufs):
        torch.cuda.synchronize()
        for b in bufs:
            assert bool(torch.isnan(b.flat.float()).all()), "rejected call wrote its output"

    # LayerNorm: C % 8 != 0, C > 1024, C <= 0 (through the raw entry points), and misaligned tensors
    from speecht5_b200 import _lib
    import ctypes as C_
    lib = _lib.load()
    st = C_.c_void_p(torch.cuda.current_stream().cuda_stream)
    for C in (12, 1032, 0, -8):
        cc = max(C, 8)
        x, g = Flat((4, cc), F32, 1.0), Flat((cc,), F32, 1.0)
        y = Flat((4, cc), F32)
        p = lambda t: C_.c_void_p(t.t.data_ptr())  # noqa: E731
        rc = lib.st5_ln_fwd(p(x), None, p(g), p(g), p(y), None, None, None, 0, 4, C, C_.c_float(EPS), C_.c_float(0.0),
                            0, 0, st)
        assert rc == -2, f"st5_ln_fwd C={C}: {rc}"
        rc = lib.st5_ln_bwd(p(x), p(x), p(g), p(g), p(g), p(y), None, None, None, None, 0, 4, C, C_.c_float(0.0), 0, 0,
                            st)
        assert rc == -2, f"st5_ln_bwd C={C}: {rc}"
        nan_all(y)
    rows, C = 8, 64
    ok = dict(x=Flat((rows, C), F32, 1.0), g=Flat((C,), F32, 1.0), s=Flat((rows, C), F32, 1.0),
              st=Flat((rows,), F32, 1.0))
    for name in ("x", "residual", "residual_f32", "gamma", "beta", "y", "y_f32", "s_out"):
        bad = Flat((rows, C) if name not in ("gamma", "beta") else (C,), F32, 1.0, off=1)  # 4 bytes off
        y, s_out, y32 = Flat((rows, C), F32), Flat((rows, C), F32), Flat((rows, C), F32)
        mean, rstd = Flat((rows,), F32), Flat((rows,), F32)
        a = dict(x=ok["x"].t, residual=None, residual_f32=None, gamma=ok["g"].t, beta=ok["g"].t, y=y.t, y_f32=None,
                 s_out=s_out.t)
        if name in ("y", "s_out"):
            bad.t.fill_(NAN)
        a[name] = bad.t
        _raises(lambda: K.ln_fwd(a["x"], a["residual"], a["gamma"], a["beta"], a["y"], a["s_out"], mean.t, rstd.t,
                                 EPS, residual_f32=a["residual_f32"], y_f32=a["y_f32"] if name == "y_f32" else y32.t),
                "st5_ln_fwd")
        nan_all(y, s_out, mean, rstd, y32)
        if name in ("y", "s_out"):
            nan_all(bad)
    for name in ("dy", "s", "gamma", "ds", "dx"):
        bad = Flat((rows, C) if name != "gamma" else (C,), F32, 1.0, off=1)
        ds, dx = Flat((rows, C), F32), Flat((rows, C), F32)
        dg, db, dxs = Flat((C,), F32), Flat((C,), F32), Flat((C,), F32)
        a = dict(dy=ok["s"].t, s=ok["s"].t, gamma=ok["g"].t, ds=ds.t, dx=dx.t)
        if name in ("ds", "dx"):
            bad.t.fill_(NAN)
        a[name] = bad.t
        _raises(lambda: K.ln_bwd(a["dy"], a["s"], ok["st"].t, ok["st"].t, a["gamma"], a["ds"], a["dx"], dg.t, db.t,
                                 dxsum=dxs.t), "st5_ln_bwd")
        nan_all(ds, dx, dg, db, dxs)

    # bn_bwd with an activation and no y_pre
    rows, C = 16, 8
    x = Flat((rows, C), F32, 1.0)
    dx, dg, db, scratch = Flat((rows, C), F32), Flat((C,), F32), Flat((C,), F32), Flat((2 * C,), F32)
    gv = Flat((C,), F32, 1.0)
    _raises(lambda: K.bn_bwd(x.t, C, x.t, C, None, gv.t, gv.t, gv.t, dx.t, C, dg.t, db.t, rows, C, "tanh", 0.0, 0, 0,
                             scratch.t), "st5_bn_bwd")
    nan_all(dx, dg, db, scratch)

    # lrelu_pad argument errors
    xb = Flat((1, 16, 8), BF16, 1.0)
    out = Flat((1, 16, 8), BF16)
    for kw in (dict(d=0, ph=0), dict(d=2, ph=2), dict(d=1, ph=-1)):
        _raises(lambda: K.lrelu_pad(xb.t, out.t, kw["d"], kw["ph"], 0, 0.1), "st5_lrelu_pad")
    x12 = Flat((1, 16, 12), BF16, 1.0)
    o12 = Flat((1, 16, 12), BF16)
    _raises(lambda: K.lrelu_pad(x12.t, o12.t, 1, 0, 0, 0.1), "st5_lrelu_pad")
    mis = Flat((1, 16, 8), BF16, 1.0, off=1)
    _raises(lambda: K.lrelu_pad(mis.t, out.t, 1, 0, 0, 0.1), "st5_lrelu_pad")
    xt = Flat((1, 16, 8), BF16, 1.0)
    _raises(lambda: K.lrelu_pad(xt.t[:, :0], out.t, 1, 0, 0, 0.1), "st5_lrelu_pad")  # T = 0
    nan_all(out, o12)

    # act_fwd / sumsq on misaligned pointers
    xa = Flat((64,), F32, 1.0, off=1)
    ya = Flat((64,), F32)
    _raises(lambda: K.act_fwd(xa.t, ya.t, "gelu"), "st5_act_fwd")
    yb = Flat((64,), F32, off=2)
    _raises(lambda: K.act_fwd(Flat((64,), F32, 1.0).t, yb.t, "gelu"), "st5_act_fwd")
    nan_all(ya, yb)
    so = Flat((1,), F32)
    _raises(lambda: K.sumsq(xa.t, so.t), "st5_sumsq")
    nan_all(so)

    # adam_step with step < 1 and no step_dev
    n = 64
    p, gg, mm, vv = (Flat((n,), F32) for _ in range(4))
    sh = Flat((n,), BF16)
    gn = torch.tensor([1.0], device="cuda")
    _raises(lambda: K.adam_step(p.t, gg.t, mm.t, vv.t, sh.t, 1e-3, 0.9, 0.98, 1e-6, 0.0, 0, gn, 1.0, 1.0),
            "st5_adam_step")
    nan_all(p, gg, mm, vv, sh)

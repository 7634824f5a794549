"""-m gpu: where every parameter gradient of a training update goes, checked elementwise against fp64 autograd.

A gradient reaches the trainer's flat fp32 buffer (trainer.FlatParams.grads) by one of several routes: a GEMM or a row
kernel that accumulates straight into the parameter's registered view (RT._static_grad, None returned to autograd) --
split-K with the L2 reduce, the S-way split + column sum, the three-pass parity product --, the bias gradient handed over
to the consuming LayerNorm (st5_ln_bwd dxsum), the relative-position table shared by every encoder layer, or a tensor
autograd adds in place into p.grad (a view of the buffer). Each route may run on the weight-gradient side stream.

Op level (Base widths, so the real split thresholds are crossed): the flat buffer is built by FlatParams itself over a
module that holds the real MultiheadAttention (fused q|k|v group) and the post-net feat_out|prob_out group; alignment gaps
are filled with NaN, every parameter region with a non-zero base (the micro-batch already accumulated), and the fp32
masters are made bf16-representable so that the bf16 shadows the GEMMs read equal the masters. After each backward
  * the parameter's region holds base + k * gradient (k backward passes) within an elementwise bound,
  * every other element -- NaN gaps and the other parameters' regions -- is bitwise unchanged,
  * every p.grad is still the flat view at fp.offsets[id(p)],
  * the calls recorded by wrapping kernels.gemm / colsum / ln_bwd / bn_bwd / l2norm_rows_bwd show the route the case is
    named for (batch count, accumulate mode, dxsum, the stream the launch was issued on).
Every case runs with and without RT.wgrad_stream (joined by RT.side_join() after backward, as B200Trainer._update does),
in throughput (bf16) and parity (fp32) mode where both exist.

Bounds (u32 = 2^-24, u16 = 2^-8): a product summed in fp32 over n terms (n = the split chunk + the number of splits + the
addition into the buffer) is within max(n, 16 sqrt(n)) u32 |A|^T |B| of the exact one -- the worst-case forward error of
an fp32 sum, never below the measured GEMM-contract constant (tests/test_gemm_contract_gpu.py) -- plus, in parity mode,
the split error of tests/conv_ref.py. An intermediate stored in bf16 (dpre after act / dropout, dH, the LayerNorm's dx)
carries its own bound e, which reaches the gradient as e^T |B|. Row kernels use the bounds of tests/rowops_ref.py,
tests/loss_ref.py and tests/attention_ref.py.

Whole update: a Base-width TTS model (2 + 2 layers, dropout 0.1, two micro-batches) through B200Trainer, eager and as a
replayed CUDA graph, against the same model run plainly (no registered buffer, every folding switch off)."""
import gc
import math
import time

import pytest
import torch
import torch.nn as nn

import attention_ref as AR
import conv_ref as CR
import dropout_ref as D
import gemm_emulator as GE
import loss_ref as LR
import rowops_ref as R

pytestmark = pytest.mark.gpu

F64 = torch.float64
U32, U16 = R.U32, R.U_BF16
TINY = R.TINY
REPORT = {}   # route / check name -> largest err / bound seen
ROUTES = {}   # (route, mode) -> number of backward passes that took it


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if REPORT:
        print("\nlargest err / bound per check:")
        for k in sorted(REPORT):
            print(f"  {k:60s} {REPORT[k]:.3g}")
    if ROUTES:
        print("routes taken (route, mode: backward passes):")
        for k in sorted(ROUTES):
            print(f"  {k[0]:40s} {k[1]:12s} {ROUTES[k]}")


@pytest.fixture(autouse=True)
def _switches():
    """The numeric mode and the backward-routing switches are process-wide: restore them whatever a case sets. Trainers,
    captured graphs and autograd graphs of a case are released here, not by a later cycle collection that could fall
    inside another test's CUDA-graph capture."""
    from speecht5_b200.ops import RT
    keep = (RT.dtype, RT.fold_residual_grad, RT.fold_bias_grad, RT.ffn_gate, RT.wgrad_splitk, RT.side_small,
            RT._seed, RT._offset)
    RT.disable_device_seed()
    RT.fold_residual_grad = RT.fold_bias_grad = RT.ffn_gate = RT.wgrad_splitk = RT.side_small = True
    yield
    (RT.dtype, RT.fold_residual_grad, RT.fold_bias_grad, RT.ffn_gate, RT.wgrad_splitk, RT.side_small,
     RT._seed, RT._offset) = keep
    RT.disable_device_seed()
    RT.wgrad_stream = None
    RT._side_keep.clear()
    RT.clear_static()
    RT.invalidate_shadows()
    gc.collect()
    torch.cuda.synchronize()


def _mode(dtype):
    return "bf16" if dtype == torch.bfloat16 else "parity"


# ------------------------------------------------------------------------------------------------------ route recorder
class Recorder:
    """Wraps (does not replace) the kernel entry points the backward routes end in and records, per call, the byte span
    of the output it writes or accumulates into, the accumulate mode, the batch count and whether the launch was issued
    on the weight-gradient side stream."""

    def __init__(self, monkeypatch):
        from speecht5_b200 import kernels as K
        self.ev = []
        for name in ("gemm", "colsum", "ln_bwd", "bn_bwd", "l2norm_rows_bwd"):
            monkeypatch.setattr(K, name, self._wrap(name, getattr(K, name)))

    def _wrap(self, name, fn):
        def call(*a, **kw):
            self.ev.append(self._event(name, a, kw))
            return fn(*a, **kw)
        return call

    @staticmethod
    def _span(t):
        if t is None:
            return None
        return (t.data_ptr(), t.data_ptr() + t.numel() * t.element_size())

    def _event(self, name, a, kw):
        from speecht5_b200.ops import RT
        cur = torch.cuda.current_stream()
        e = dict(kind=name, side=RT.wgrad_stream is not None and cur.cuda_stream == RT.wgrad_stream.cuda_stream)
        if name == "gemm":
            e.update(out=self._span(a[2]), acc=int(kw.get("accumulate", 0)), nb1=kw.get("nb1", 1), nb2=kw.get("nb2", 1))
        elif name == "colsum":
            e.update(out=self._span(a[1]), acc=bool(kw.get("accumulate", a[3] if len(a) > 3 else False)), src=a[0])
        elif name == "ln_bwd":
            e.update(out=self._span(kw.get("dxsum")), dgamma=self._span(a[7]), dbeta=self._span(a[8]))
        elif name == "bn_bwd":
            e.update(out=None, dgamma=self._span(a[10]), dbeta=self._span(a[11]))
        else:
            e.update(out=self._span(a[3]), acc=bool(kw.get("accumulate", False)))
        return e

    def into(self, kind, span, key="out"):
        return [e for e in self.ev if e["kind"] == kind and e.get(key) is not None
                and span[0] <= e[key][0] and e[key][1] <= span[1]]


def _region(fp, params):
    """Byte span of the (contiguous) flat-gradient region of a parameter group."""
    o = fp.offsets[id(params[0])]
    n = 0
    for p in params:
        assert fp.offsets[id(p)] == o + n, "a fused group is not contiguous in the flat buffer"
        n += p.numel()
    base = fp.grads.data_ptr()
    return (base + 4 * o, base + 4 * (o + n))


def _route(rec, fp, route, params, side, mode, **kw):
    """Assert that the gradient of `params` took `route` in the backward pass `rec` recorded."""
    span = _region(fp, params)
    flat = (fp.grads.data_ptr(), fp.grads.data_ptr() + 4 * fp.numel)
    if route == "splitk_l2":
        ev = rec.into("gemm", span)
        assert len(ev) == 1 and ev[0]["acc"] == 2 and ev[0]["nb1"] == kw["S"], ev
        assert ev[0]["side"] == side, ev
    elif route == "s_split_colsum":
        ev = rec.into("colsum", span)
        assert len(ev) == 1 and ev[0]["acc"], ev
        parts = [e for e in rec.ev if e["kind"] == "gemm" and e["nb1"] == kw["S"] and not (flat[0] <= e["out"][0] < flat[1])]
        assert parts, "no S-way partial product"
        assert not rec.into("gemm", span)
    elif route == "parity_mm":
        ev = rec.into("gemm", span)
        assert len(ev) == 3 and all(e["acc"] == 1 and e["nb1"] == 1 for e in ev), ev
    elif route == "colsum":
        ev = rec.into("colsum", span)
        assert len(ev) == 1 and ev[0]["acc"], ev
        assert ev[0]["side"] == side, ev
    elif route == "ln_dxsum":
        ev = rec.into("ln_bwd", span)
        assert len(ev) == 1 and ev[0]["out"] == span, ev
        assert not rec.into("colsum", span) and not rec.into("gemm", span)
    elif route in ("ln_direct", "bn_direct"):
        g, b = params
        ev = rec.into(route[:2] + "_bwd", _region(fp, [g]), key="dgamma")
        assert len(ev) == 1 and ev[0]["dgamma"] == _region(fp, [g]) and ev[0]["dbeta"] == _region(fp, [b]), ev
    elif route == "l2_accumulate":
        ev = rec.into("l2norm_rows_bwd", span)
        assert len(ev) == 1 and ev[0]["acc"], ev
    elif route == "table_head_major":
        ev = rec.into("gemm", span)
        assert len(ev) == kw["calls"] and all(e["acc"] == 2 and e["nb1"] == kw["H"] and e["nb2"] == kw["S"]
                                              for e in ev), ev
        assert all(e["side"] == side for e in ev), ev
    elif route == "autograd":  # the Function returned the gradient: nothing writes the region before AccumulateGrad
        assert not any(rec.into(k, span) for k in ("gemm", "colsum", "ln_bwd", "l2norm_rows_bwd"))
    else:
        raise AssertionError(route)
    ROUTES[(route, mode)] = ROUTES.get((route, mode), 0) + 1


# ------------------------------------------------------------------------------------------------------ bounds
def _prod(mag, n, parity):
    """Forward-error bound of a product accumulated in fp32 over n terms; parity mode adds the bf16 split."""
    c = max(n, CR.C_ACC * math.sqrt(n)) * U32
    if parity:
        return c * (1 + 2.02 * U16) * mag + (CR.SPLIT + 3 * U32) * mag
    return c * mag


def _colsum_bound(v, e):
    return R.C_COL * U32 * v.abs().sum(0) + e.sum(0) + TINY


# ------------------------------------------------------------------------------------------------------ the parameters
class Holder(nn.Module):
    """The parameters under test, in the modules the model uses (so FlatParams forms the same fused groups)."""

    def __init__(self):
        super().__init__()
        from speecht5_b200.models.modules.transformer import MultiheadAttention
        self.attn = MultiheadAttention(768, 12, self_attention=True)
        self.lin = nn.Linear(768, 768)
        self.fc1 = nn.Linear(768, 3072)
        self.fc2 = nn.Linear(3072, 768)
        self.ln = nn.LayerNorm(768)
        self.speech_decoder_postnet = nn.Module()
        self.speech_decoder_postnet.feat_out = nn.Linear(768, 160)
        self.speech_decoder_postnet.prob_out = nn.Linear(768, 2)
        self.bn = nn.BatchNorm1d(256)
        self.table = nn.Embedding(320, 64)
        self.cls = nn.Parameter(torch.randn(200, 256))
        with torch.no_grad():
            for m in (self.ln, self.bn):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.5, 0.5)
            for lin in (self.attn.q_proj, self.attn.k_proj, self.attn.v_proj, self.attn.out_proj, self.lin, self.fc1,
                        self.fc2, self.speech_decoder_postnet.feat_out, self.speech_decoder_postnet.prob_out):
                lin.bias.uniform_(-0.3, 0.3)
            self.table.weight.mul_(0.3)


class Flat:
    """The parameters under test with (registered=True) or without the trainer's flat buffers."""

    def __init__(self, dev, registered):
        from speecht5_b200.ops import RT
        from speecht5_b200.trainer import FlatParams
        torch.manual_seed(0)
        self.h = Holder().to(dev)
        self.params = list(self.h.parameters())
        self.fp = None
        if not registered:
            RT.clear_static()
            with torch.no_grad():
                for p in self.params:
                    p.copy_(p.bfloat16().float())
                    p.grad = None
            RT.invalidate_shadows()
            return
        fp = self.fp = FlatParams(self.h)
        with torch.no_grad():
            fp.flat.copy_(fp.flat.bfloat16().float())  # masters = their bf16 shadows
        fp.refresh_shadow()
        owned = torch.zeros(fp.numel, dtype=torch.bool, device=dev)
        g = torch.Generator(device=dev).manual_seed(5)
        base = torch.full((fp.numel,), float("nan"), device=dev)
        for p in self.params:
            o, n = fp.offsets[id(p)], p.numel()
            owned[o:o + n] = True
            mag = torch.rand(n, device=dev, generator=g) + 1.0
            base[o:o + n] = torch.where(torch.rand(n, device=dev, generator=g) < 0.5, -mag, mag)
        assert not bool(owned.all()), "the layout has no alignment gap to fill with NaN"
        fp.grads.copy_(base)
        self.base = base.clone()

    def check(self, name, expect, k, report=REPORT):
        """expect: [(params of one contiguous group, fp64 gradient of ONE backward, its bound)] after k backwards."""
        if self.fp is None:
            for params, ref, bnd in expect:
                got = torch.cat([p.grad.reshape(-1) for p in params])
                ref, bnd = ref.to(got.device), bnd.to(got.device)
                R.check(f"{name}: {'|'.join(_pname(self.h, p) for p in params)}", got, k * ref.reshape(-1),
                        k * bnd.reshape(-1) + k * U32 * ref.abs().reshape(-1), report)
            return
        fp = self.fp
        want = self.base.double()
        bound = torch.zeros_like(want)
        mine = torch.zeros(fp.numel, dtype=torch.bool, device=want.device)
        for params, ref, bnd in expect:
            o = fp.offsets[id(params[0])]
            n = sum(p.numel() for p in params)
            assert _region(fp, params)  # (contiguity)
            want[o:o + n] = want[o:o + n] + k * ref.reshape(-1).to(want.device)
            bound[o:o + n] = k * bnd.reshape(-1).to(want.device) + (k + 1) * U32 * (want[o:o + n].abs()
                                                                                    + self.base[o:o + n].double().abs())
            mine[o:o + n] = True
        for params, _, _ in expect:
            o = fp.offsets[id(params[0])]
            n = sum(p.numel() for p in params)
            R.check(f"{name}: {'|'.join(_pname(self.h, p) for p in params)}", fp.grads[o:o + n], want[o:o + n],
                    bound[o:o + n], report)
        rest = ~mine
        same = fp.grads.view(torch.int32)[rest] == self.base.view(torch.int32)[rest]
        if not bool(same.all()):
            idx = int(torch.nonzero(rest)[int(torch.nonzero(~same)[0])])
            owner = [(_pname(self.h, p), fp.offsets[id(p)]) for p in self.params
                     if fp.offsets[id(p)] <= idx < fp.offsets[id(p)] + p.numel()]
            raise AssertionError(f"{name}: flat element {idx} outside the expected regions changed "
                                 f"(owner {owner or 'alignment gap'}): {float(self.base[idx])} -> {float(fp.grads[idx])}")
        for p in self.params:
            assert p.grad is not None, _pname(self.h, p)
            assert p.grad.data_ptr() == fp.grads.data_ptr() + 4 * fp.offsets[id(p)] and p.grad.shape == p.shape, \
                f"{name}: p.grad of {_pname(self.h, p)} is no longer its flat view"


def _pname(h, p):
    for n, q in h.named_parameters():
        if q is p:
            return n
    return "?"


def _backward(side, outs, grads):
    """One backward pass, with the weight-gradient side stream as B200Trainer._update opens and joins it."""
    from speecht5_b200.ops import RT
    RT.wgrad_stream = torch.cuda.Stream() if side else None
    try:
        torch.autograd.backward(outs, grads)
        RT.side_join()
    finally:
        RT.wgrad_stream = None
    torch.cuda.synchronize()


def _keep_gemm(M, N, p, seed, off, dev):
    return GE.gemm_keep(M, N, 1, p, seed, off).reshape(M, N).to(dev)


def _keep_rows(rows, C, p, seed, off, dev):
    return R.keep((rows, C), p, seed, off).to(dev)


def _saved(y):
    """(saved tensors, meta) of the Function that produced y -- read before backward frees them."""
    return y.grad_fn.saved_tensors, y.grad_fn.meta


def _ln_ref(sv, gy, dtype):
    """fp64 backward of ResidualLayerNormFn from what its forward saved (s, mean, rstd) and its dropout draw."""
    (s, mean, rstd, gamma), meta = sv
    drop_p, off, seed = meta[:3]
    C = s.shape[-1]
    rows = s.numel() // C
    kp = _keep_rows(rows, C, drop_p, seed, off, s.device).to(F64) if drop_p > 0 else None
    b = R.ln_backward(gy.reshape(rows, C), s.reshape(rows, C), mean, rstd, gamma.detach(), kp=kp,
                      dscale=D.drop_scale(drop_p) if drop_p > 0 else 1.0)
    return b, R.ln_backward_bounds(b, R.unit(dtype))


def _act_dpre(g, pre, act, u):
    """dpre = g act'(pre) and its bound (pre as the forward stored it)."""
    if act is None:
        return g, u * g.abs()
    return R.act_bwd_bound(g, pre, act, u)


# ------------------------------------------------------------------------------------------------------ LinearFn cases
LIN_CASES = ["qkv_2304x768", "splitk_s3", "out_proj_handover", "out_proj_handover_unregistered", "postnet_feat_prob",
             "gelu_dropout", "passthrough_both", "passthrough_alias_only", "no_dx"]


def _lin_setup(case, h):
    a = h.attn
    if case == "qkv_2304x768":
        return (a.q_proj.weight, a.k_proj.weight, a.v_proj.weight), (a.q_proj.bias, a.k_proj.bias, a.v_proj.bias), 4, 384
    if case.startswith("out_proj"):
        return (a.out_proj.weight,), (a.out_proj.bias,), 4, 384
    if case == "postnet_feat_prob":
        po = h.speech_decoder_postnet
        return (po.feat_out.weight, po.prob_out.weight), (po.feat_out.bias, po.prob_out.bias), 4, 512
    return (h.lin.weight,), (h.lin.bias,), 4, 384


@pytest.mark.parametrize("side", [False, True], ids=["main", "side"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "parity"])
@pytest.mark.parametrize("case", LIN_CASES)
def test_linear_gradient_routes(cuda, monkeypatch, case, dtype, side):
    from speecht5_b200 import ops
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    parity = dtype == torch.float32
    mode = _mode(dtype)
    u = R.unit(dtype)
    fl = Flat(cuda, registered=not case.endswith("unregistered"))
    h, fp = fl.h, fl.fp
    ws, bs, B, T = _lin_setup(case, h)
    N, Kd = sum(w.shape[0] for w in ws), ws[0].shape[1]
    M = B * T
    handover = case.startswith("out_proj")
    act = "gelu" if case == "gelu_dropout" else None
    drop_p = 0.1 if case == "gelu_dropout" else 0.0
    gen = torch.Generator(device=cuda).manual_seed(11)
    x0 = torch.randn(B, T, Kd, device=cuda, generator=gen).to(dtype)
    gy = torch.randn(B, T, N, device=cuda, generator=gen).to(dtype)
    res0 = torch.randn(B, T, N, device=cuda, generator=gen).to(dtype)
    gr = torch.randn(B, T, Kd, device=cuda, generator=gen).to(dtype)
    rec = Recorder(monkeypatch)
    for k in (1, 2):
        rec.ev.clear()
        RT.manual_seed(3)
        x = x0.clone().requires_grad_()
        if handover:
            r = res0.clone().requires_grad_()
            o = ops.linear(x, ws, bs, bias_grad_by_consumer=True)
            sv_lin = _saved(o)
            y = ops.residual_layer_norm(o, r, h.ln, drop_p=0.1)
            lin_out, sv_ln = o, _saved(y)
            _backward(side, [y], [gy])
        elif case == "postnet_feat_prob":
            y = ops.linear(x, ws, bs, out_dtype=torch.float32)
            lin_out, sv_lin = y, _saved(y)
            _backward(side, [y], [gy.float()])
        elif case.startswith("passthrough"):
            y, x_pt = ops.linear(x, ws, bs, passthrough=True)
            lin_out, sv_lin = y, _saved(y)
            if case == "passthrough_both":
                _backward(side, [y, x_pt], [gy, gr])
            else:
                _backward(side, [x_pt], [gr])
        else:
            y = ops.linear(x, ws, bs, act=act, drop_p=drop_p, need_dx=case != "no_dx")
            lin_out, sv_lin = y, _saved(y)
            _backward(side, [y], [gy])
        # ---- fp64 reference from the operands the kernels read
        off, seed = sv_lin[1][6], sv_lin[1][15]
        x64 = x0.reshape(M, Kd).double()
        W64 = torch.cat([w.detach() for w in ws]).double()
        if handover:
            lb, lbb = _ln_ref(sv_ln, gy, dtype)
            g, eg = lb["dx"], lbb["dx"]
        elif case == "passthrough_alias_only":
            g, eg = torch.zeros(M, N, dtype=F64, device=cuda), torch.zeros(M, N, dtype=F64, device=cuda)
        else:
            g, eg = gy.reshape(M, N).double(), torch.zeros(M, N, dtype=F64, device=cuda)
        if drop_p > 0:
            g = g * _keep_gemm(M, N, drop_p, seed, off, cuda) * D.drop_scale(drop_p)
        pre = sv_lin[0][1]
        if act is not None:
            dpre, edp = _act_dpre(g, pre[:, :N].double(), ops._resolve_act(act, dtype), u)
        else:
            dpre, edp = g, eg
        S = {"qkv_2304x768": 1, "postnet_feat_prob": 8}.get(case, 3) if not parity else 1
        n_w = M // S + S + 1
        dW = dpre.t() @ x64
        bW = _prod(dpre.abs().t() @ x64.abs(), n_w, parity) + edp.t() @ x64.abs()
        expect = [(list(ws), dW, bW)]
        db = dpre.sum(0)
        if handover:
            expect += [(list(bs), lb["dxsum"], lbb["dxsum"]), ([h.ln.weight], lb["dgamma"], lbb["dgamma"]),
                       ([h.ln.bias], lb["dbeta"], lbb["dbeta"])]
        else:
            expect.append((list(bs), db, _colsum_bound(dpre, edp)))
        fl.check(f"{case}[{mode},{'side' if side else 'main'}]", expect, k)
        # ---- input gradient (the residual branch folded into the dx GEMM for passthrough)
        if case == "no_dx":
            assert x.grad is None
        else:
            dx = dpre @ W64
            bx = _prod(dpre.abs() @ W64.abs(), N, parity) + edp @ W64.abs()
            if case.startswith("passthrough"):
                dx = dx + gr.reshape(M, Kd).double()
                bx = bx + U32 * gr.reshape(M, Kd).double().abs()
            R.check(f"{case}[{mode}] dx", x.grad.reshape(M, Kd), dx, bx + u * dx.abs() + TINY, REPORT)
            if handover:
                R.check(f"{case}[{mode}] d residual", r.grad.reshape(M, N), lb["ds"], lbb["ds"], REPORT)
        # ---- the route
        if fp is not None:
            if parity:
                _route(rec, fp, "parity_mm", list(ws), side, mode)
            elif case == "postnet_feat_prob":
                _route(rec, fp, "s_split_colsum", list(ws), side, mode, S=8)
            else:
                _route(rec, fp, "splitk_l2", list(ws), side, mode, S=S)
            if handover:
                _route(rec, fp, "ln_dxsum", list(bs), side, mode)
                _route(rec, fp, "ln_direct", [h.ln.weight, h.ln.bias], side, mode)
            else:
                _route(rec, fp, "colsum", list(bs), side, mode)


# ------------------------------------------------------------------------------------------------------ FFNFn
@pytest.mark.parametrize("side", [False, True], ids=["main", "side"])
@pytest.mark.parametrize("mode", ["bf16_gate", "bf16_nogate", "parity"])
def test_ffn_gradient_routes(cuda, monkeypatch, mode, side):
    """fc1 (768 -> 3072, GELU, dropout 0.1) + fc2 feeding the LayerNorm that takes fc2's bias gradient over, the block
    input passed through so that the residual branch's gradient is added in the dx GEMM; with the backward gate fc1
    stores (keep * scale * gelu'(pre), replacing act' and the mask in the dH epilogue) and without it."""
    from speecht5_b200 import ops
    from speecht5_b200.ops import RT
    dtype = torch.float32 if mode == "parity" else torch.bfloat16
    parity = dtype == torch.float32
    RT.dtype = dtype
    RT.ffn_gate = mode == "bf16_gate"
    u = R.unit(dtype)
    fl = Flat(cuda, registered=True)
    h, fp = fl.h, fl.fp
    B, T, Dm, Fd = 4, 384, 768, 3072
    M = B * T
    gen = torch.Generator(device=cuda).manual_seed(12)
    x0 = torch.randn(B, T, Dm, device=cuda, generator=gen).to(dtype)
    gy = torch.randn(B, T, Dm, device=cuda, generator=gen).to(dtype)
    rec = Recorder(monkeypatch)
    for k in (1, 2):
        rec.ev.clear()
        RT.manual_seed(4)
        x = x0.clone().requires_grad_()
        o, x_pt = ops.ffn(x, h.fc1, h.fc2, "gelu", drop_a=0.1, passthrough=True, bias_grad_by_consumer=True)
        y = ops.residual_layer_norm(o, x_pt, h.ln, drop_p=0.1, stream=True)
        (x2, hs, pre_or_gate), meta = _saved(o)
        sv_ln = _saved(y)
        _backward(side, [y], [gy])
        act, drop_a, off_a, seed = meta[6], meta[7], meta[8], meta[11]
        assert (act == "gate") == (mode == "bf16_gate")
        lb, lbb = _ln_ref(sv_ln, gy, dtype)
        dO, eO = lb["dx"], lbb["dx"]
        x64, h64 = x0.reshape(M, Dm).double(), hs.double()
        W1, b1, W2 = h.fc1.weight.detach().double(), h.fc1.bias.detach().double(), h.fc2.weight.detach().double()
        keep = _keep_gemm(M, Fd, drop_a, seed, off_a, cuda).to(F64) * D.drop_scale(drop_a)
        dW2 = dO.t() @ h64
        bW2 = _prod(dO.abs().t() @ h64.abs(), M + 2, parity) + eO.t() @ h64.abs()
        dHl = dO @ W2
        eHl = _prod(dO.abs() @ W2.abs(), Dm, parity) + eO @ W2.abs()
        if act == "gate":
            # the stored gate against keep * scale * gelu_tanh'(pre) from the fp64 pre-activation
            pre64 = x64 @ W1.t() + b1
            epre = _prod(x64.abs() @ W1.abs().t(), Dm, False) + U32 * pre64.abs()
            dref, ed = R.act_bwd_bound(torch.ones_like(pre64), pre64, "gelu_tanh", 0.0)
            gate = keep * dref
            R.check(f"ffn[{mode}] gate", pre_or_gate.double(), gate, keep * (CR.A2 * epre + ed) + U16 * gate.abs() + TINY,
                    REPORT)
            gs = pre_or_gate.double()
            dH = dHl * gs
            eH = eHl * gs.abs() + 2 * U32 * dH.abs() + u * dH.abs() + TINY
        else:
            dH, eH = R.act_bwd_bound(dHl * keep, pre_or_gate.double(), ops._resolve_act("gelu", dtype), u)
            eH = eH + eHl * keep * R.act_grad(pre_or_gate.double(), ops._resolve_act("gelu", dtype)).abs()
        dW1 = dH.t() @ x64
        bW1 = _prod(dH.abs().t() @ x64.abs(), M + 2, parity) + eH.t() @ x64.abs()
        # fc1's bias gradient is the column sum of the stored dH (the tensor the column-sum kernel read): check that tensor
        # against the fp64 dH, and the bias against the exact sum of it
        src = [e["src"] for e in rec.into("colsum", _region(fp, [h.fc1.bias]))]
        assert len(src) == 1, "fc1's bias gradient did not come from one column sum"
        R.check(f"ffn[{mode}] dH as stored", src[0], dH, eH, REPORT)
        dHs = src[0].double()
        expect = [([h.fc1.weight], dW1, bW1), ([h.fc1.bias], dHs.sum(0), _colsum_bound(dHs, torch.zeros_like(dHs))),
                  ([h.fc2.weight], dW2, bW2), ([h.fc2.bias], lb["dxsum"], lbb["dxsum"]),
                  ([h.ln.weight], lb["dgamma"], lbb["dgamma"]), ([h.ln.bias], lb["dbeta"], lbb["dbeta"])]
        fl.check(f"ffn[{mode},{'side' if side else 'main'}]", expect, k)
        dx = dH @ W1 + lb["ds"]
        bx = _prod(dH.abs() @ W1.abs(), Fd, parity) + eH @ W1.abs() + lbb["ds"] + (U32 + u) * dx.abs() + TINY
        R.check(f"ffn[{mode}] dx (+ folded residual gradient)", x.grad.reshape(M, Dm), dx, bx, REPORT)
        for w in (h.fc1.weight, h.fc2.weight):
            _route(rec, fp, "parity_mm" if parity else "splitk_l2", [w], side, mode, S=1)
        _route(rec, fp, "colsum", [h.fc1.bias], side, mode)
        _route(rec, fp, "ln_dxsum", [h.fc2.bias], side, mode)
        _route(rec, fp, "ln_direct", [h.ln.weight, h.ln.bias], side, mode)


# ------------------------------------------------------------------------------------------------------ row kernels
@pytest.mark.parametrize("side", [False, True], ids=["main", "side"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "parity"])
@pytest.mark.parametrize("case", ["layer_norm", "batch_norm_tanh_dropout", "l2norm_class_weight"])
def test_row_kernel_gradient_routes(cuda, monkeypatch, case, dtype, side):
    """dgamma / dbeta of ResidualLayerNormFn and BatchNormActFn added by the kernels straight into the registered views;
    the s2c class weight's gradient accumulated by st5_l2norm_rows_bwd into its view (grad_key)."""
    from speecht5_b200 import ops
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    mode = _mode(dtype)
    u = R.unit(dtype)
    fl = Flat(cuda, registered=True)
    h, fp = fl.h, fl.fp
    gen = torch.Generator(device=cuda).manual_seed(13)
    C = 768 if case == "layer_norm" else 256
    x0 = torch.randn(6, 211, C, device=cuda, generator=gen).to(dtype)
    r0 = torch.randn(6, 211, C, device=cuda, generator=gen).to(dtype)
    gy = torch.randn(6, 211, C, device=cuda, generator=gen).to(dtype)
    gcls = torch.randn(200, 256, device=cuda, generator=gen)
    rec = Recorder(monkeypatch)
    rows = 6 * 211
    for k in (1, 2):
        rec.ev.clear()
        RT.manual_seed(5)
        x = x0.clone().requires_grad_()
        if case == "layer_norm":
            y = ops.residual_layer_norm(x, r0, h.ln, drop_p=0.1)
            sv = _saved(y)
            _backward(side, [y], [gy])
            lb, lbb = _ln_ref(sv, gy, dtype)
            expect = [([h.ln.weight], lb["dgamma"], lbb["dgamma"]), ([h.ln.bias], lb["dbeta"], lbb["dbeta"])]
            route = ("ln_direct", [h.ln.weight, h.ln.bias])
        elif case == "batch_norm_tanh_dropout":
            y = ops.batch_norm_act(x, h.bn, training=True, act="tanh", drop_p=0.1)
            (xs, y_pre, gamma, mean, rstd), meta = _saved(y)
            _backward(side, [y], [gy])
            _, drop_p, off, seed = meta[:4]
            kp = _keep_rows(rows, C, drop_p, seed, off, cuda).to(F64)
            b = R.bn_backward(gy.reshape(rows, C), xs.reshape(rows, C), y_pre.reshape(rows, C), gamma.detach(), mean,
                              rstd, act_name="tanh", kp=kp, dscale=D.drop_scale(drop_p))
            bb = R.bn_backward_bounds(b, u)
            expect = [([h.bn.weight], b["dgamma"], bb["dgamma"]), ([h.bn.bias], b["dbeta"], bb["dbeta"])]
            route = ("bn_direct", [h.bn.weight, h.bn.bias])
        else:
            yn = ops.l2_normalize_rows(h.cls, grad_key=("lin", id(h.cls)))
            (ys, nrm), _ = _saved(yn)
            _backward(side, [yn], [gcls])
            dref, e = LR.l2norm_bwd(gcls, ys, nrm)
            expect = [([h.cls], dref, e)]
            route = ("l2_accumulate", [h.cls])
        fl.check(f"{case}[{mode},{'side' if side else 'main'}]", expect, k)
        _route(rec, fp, route[0], route[1], side, mode)


# ------------------------------------------------------------------------------------------------------ shared table
@pytest.mark.parametrize("side", [False, True], ids=["main", "side"])
@pytest.mark.parametrize("case", ["head_major", "unregistered", "b_x_h"])
def test_relative_position_table_shared_by_three_layers(cuda, monkeypatch, case, side):
    """One relative-position table used by three self-attention calls (three encoder layers): the head-major route adds
    each layer's contribution into the registered view (split over rows, on the side stream when it is open); without a
    registered view autograd sums the three returned tensors; the B x H route (RT.wgrad_splitk off) returns each layer's
    table gradient and autograd adds it in place into p.grad, the flat view."""
    from speecht5_b200 import ops
    from speecht5_b200.ops import RT
    RT.dtype = torch.bfloat16
    RT.wgrad_splitk = case != "b_x_h"
    fl = Flat(cuda, registered=case != "unregistered")
    h, fp = fl.h, fl.fp
    B, H, T, d, maxpos, L = 8, 12, 160, 768, 160, 3
    sc = 0.125
    gen = torch.Generator(device=cuda).manual_seed(14)
    qkv0 = [(torch.randn(B, T, 3 * d, device=cuda, generator=gen) * 0.8).bfloat16() for _ in range(L)]
    dO = [torch.randn(B, T, d, device=cuda, generator=gen).bfloat16() for _ in range(L)]
    lens = torch.tensor([T, T - 13, T - 40, T, T - 1, T - 77, T, T - 5], device=cuda)
    key_pad = torch.arange(T, device=cuda)[None, :] >= lens[:, None]
    table = h.table.weight
    # fp64 reference on the host, layer by layer
    ref = torch.zeros(2 * maxpos, 64, dtype=F64)
    bnd = torch.zeros_like(ref)
    pe = table.detach().cpu()
    n_acc = B * T * H + 2 * L + 2
    for l in range(L):
        q, k_, v = [t.reshape(B, T, H, 64).transpose(1, 2) for t in qkv0[l].cpu().double().split(d, dim=-1)]
        f = AR.forward(q, k_, v, scale=sc, pe=pe, maxpos=maxpos, key_pad=key_pad.cpu())
        g = AR.backward(f, dO[l].cpu().double().reshape(B, T, H, 64).transpose(1, 2))
        b = AR.bounds(f, g, u=AR.U_BF16, C=AR.C_BF16)
        ref += g["dPE"]
        mag = sc * torch.einsum("bhir,bhic->rc", g["dQP"].abs(), q.abs())
        bnd += b["dPE"] + U16 * mag + n_acc * U32 * (mag + sc * torch.einsum("bhir,bhic->rc", b["dQP"], q.abs()))
    rec = Recorder(monkeypatch)
    for k in (1, 2):
        rec.ev.clear()
        RT.manual_seed(6)
        outs = []
        for l in range(L):
            out, _ = ops.attention(qkv0[l].clone().requires_grad_(), None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=sc,
                                   pe_k=table, maxpos=maxpos, key_pad=key_pad)
            outs.append(out)
        _backward(side, outs, dO)
        fl.check(f"table[{case},{'side' if side else 'main'}]", [([table], ref, bnd)], k)
        if fp is not None:
            if case == "head_major":
                _route(rec, fp, "table_head_major", [table], side, "bf16", calls=L, H=H, S=2)
            else:
                _route(rec, fp, "autograd", [table], side, "bf16")
        else:
            ROUTES[("table_unregistered", "bf16")] = ROUTES.get(("table_unregistered", "bf16"), 0) + 1


# ------------------------------------------------------------------------------------------------------ whole update
WHOLE = dict(encoder_layers=2, decoder_layers=2, dropout=0.1, attention_dropout=0.1, activation_dropout=0.1,
             encoder_layerdrop=0.0, decoder_layerdrop=0.0, bert_init=True)
# per-parameter relative difference of the trainer's gradients from the plain model's: at most this, or three times the
# plain model's own run-to-run spread where that is larger (bf16 post-net BatchNorm biases: sums that cancel, over
# activations whose bf16 roundings follow the atomic order of the forward statistics). Parity mode: ~2^-16 products.
WHOLE_TOL = {torch.bfloat16: 2e-2, torch.float32: 1e-4}
# post-net output and losses of the trainer against the plain model (fp32 atomic order of the BatchNorm statistics)
BN_ATOMIC_TOL = {torch.bfloat16: 2e-3, torch.float32: 1e-5}


def _whole_model(dev, dtype):
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    RT.dtype = dtype
    RT.clear_static()
    torch.manual_seed(0)
    args = make_args("t5_transformer_base_asr", **WHOLE)
    task = SpeechT5Task(args)
    model = task.build_model(args).to(dev).train()
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(p.bfloat16().float())  # the bf16 shadows of both arms equal the fp32 masters
    RT.invalidate_shadows()
    return task, model, SpeechT5Criterion(task, use_guided_attn_loss=True)


def _plain_arm(dev, dtype, mbs, seed, heads):
    """No trainer, nothing registered, every backward folding switch off; gradients summed over the micro-batches. The
    attention backward gets the trainer's hint that the guided-attention loss differentiates only the first `heads`
    heads of the returned maps (RT.probs_grad_heads): that is a property of the criterion, not a gradient route, and it
    changes the fp32 summation order of the attention's row constants."""
    from speecht5_b200.ops import RT
    task, model, crit = _whole_model(dev, dtype)
    RT.fold_residual_grad = RT.fold_bias_grad = RT.ffn_gate = RT.wgrad_splitk = False
    RT.probs_grad_heads = heads
    RT.disable_device_seed()
    RT.manual_seed(seed)
    outs, losses = [], []
    hook = model.register_forward_hook(lambda m, i, o: outs.append((o[0].detach().clone(), o[1].detach().clone())))
    try:
        for mb in mbs:
            loss = task.train_step(mb, model, crit, None, 0)[0]
            losses.append(torch.as_tensor(loss, dtype=torch.float32, device=dev).detach().reshape(()).clone())
    finally:
        hook.remove()
        RT.fold_residual_grad = RT.fold_bias_grad = RT.ffn_gate = RT.wgrad_splitk = True
        RT.probs_grad_heads = 0
    torch.cuda.synchronize()
    return {n: (p.grad.detach().clone() if p.grad is not None else None) for n, p in model.named_parameters()}, outs, \
        torch.stack(losses)


def _trainer_arm(dev, dtype, mbs, graph, monkeypatch):
    from speecht5_b200.ops import RT
    from speecht5_b200.trainer import B200Trainer
    task, model, crit = _whole_model(dev, dtype)
    RT.disable_device_seed()
    tr = B200Trainer(model, crit, task, lr=0.0, use_cuda_graph=graph)
    assert RT.probs_grad_heads > 0  # (guided attention on: the hint _plain_arm repeats)
    seed = int(tr.state_dict()["dropout_seed"])
    RT.manual_seed(seed)
    outs = []
    hook = model.register_forward_hook(lambda m, i, o: outs.append((o[0].detach().clone(), o[1].detach().clone())))
    rec = Recorder(monkeypatch) if not graph else None
    try:
        losses = tr.train_step(mbs)[0]
    finally:
        hook.remove()
    torch.cuda.synchronize()
    return tr, model, seed, outs, losses.float().reshape(-1).clone(), rec


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "parity"])
def test_whole_update_gradients_equal_the_plain_model(cuda, monkeypatch, dtype):
    """Base widths, 2 + 2 layers, TTS with guided attention, dropout 0.1, two micro-batches of 8 utterances x 160 tokens
    x 600 frames. E: B200Trainer, eager update; G (bf16): the same update as a replayed CUDA graph. Each against P, the
    plain model at the same dropout seed. The forward is the same computation in E and P (the switches that differ act in
    backward only): the decoder output agrees bit for bit, the post-net output and the losses to the fp32 atomic order of
    the post-net's BatchNorm statistics; the gradients differ only by summation order and roundings."""
    from speecht5_b200.data import synthetic_tts_batch
    from speecht5_b200.trainer import _to_device
    from speecht5_b200.ops import RT
    t0 = time.time()
    mbs = [_to_device(synthetic_tts_batch(8, 160, 600, seed=30 + i), cuda) for i in range(2)]
    arms = [("E", False)] + ([("G", True)] if dtype == torch.bfloat16 else [])
    mode = _mode(dtype)
    for arm, graph in arms:
        tr, model, seed, outs_t, losses_t, rec = _trainer_arm(cuda, dtype, mbs, graph, monkeypatch)
        heads = RT.probs_grad_heads
        fp = tr.fp
        names = {id(p): n for n, p in model.named_parameters()}
        grads_t = {names[id(p)]: fp.grads[fp.offsets[id(p)]:fp.offsets[id(p)] + p.numel()].view(p.shape).clone()
                   for p in fp.params}
        gnorm_sq = float(tr.gnorm_sq)
        owned = torch.zeros(fp.numel, dtype=torch.bool, device=cuda)
        for p in fp.params:
            owned[fp.offsets[id(p)]:fp.offsets[id(p)] + p.numel()] = True
        assert float(fp.grads[~owned].abs().max()) == 0.0, f"{arm}: the flat buffer's padding was written"
        grads_ref = {n: p.grad for n, p in model.named_parameters()}  # (p.grad: still the flat view)
        for p in fp.params:
            assert p.grad is not None and p.grad.data_ptr() == fp.grads.data_ptr() + 4 * fp.offsets[id(p)], names[id(p)]
        del tr, model, grads_ref
        RT_reset()
        grads_p, outs_p, losses_p = _plain_arm(cuda, dtype, mbs, seed, heads)
        # the plain model against itself: its run-to-run spread (forward BatchNorm statistics and backward parameter
        # sums are fp32 atomics) is the floor below which the trainer's routes cannot be told apart from it
        grads_q = _plain_arm(cuda, dtype, mbs, seed, heads)[0]
        # the decoder output before the post-net is the same computation in both arms: bit for bit; the post-net's
        # BatchNorm statistics are column sums that st5_bn_fwd adds with fp32 atomics (order varies from run to run),
        # so the refined output and the losses computed from it agree to that reduction's rounding only
        if not graph:
            assert len(outs_t) == len(outs_p) == 2
            for (b_t, a_t), (b_p, a_p) in zip(outs_t, outs_p):
                assert torch.equal(b_t, b_p), f"{arm}: decoder output differs from the plain model's"
                ea = float((a_t.double() - a_p.double()).norm() / a_p.double().norm())
                REPORT[f"whole update {arm}[{mode}] post-net output rel err"] = max(
                    ea, REPORT.get(f"whole update {arm}[{mode}] post-net output rel err", 0.0))
                assert ea <= BN_ATOMIC_TOL[dtype], (arm, ea)
        el = float(((losses_t.double() - losses_p.double()).abs() / losses_p.double().abs()).max())
        REPORT[f"whole update {arm}[{mode}] loss rel err"] = el
        assert el <= BN_ATOMIC_TOL[dtype], (arm, losses_t, losses_p)
        gmax = max(float(g.norm()) for g in grads_p.values() if g is not None)
        worst, worst_name, worst_ratio, sq = 0.0, None, 0.0, 0.0
        for n, gp in grads_p.items():
            gt = grads_t[n]
            if gp is None:
                assert float(gt.abs().max()) == 0.0, f"{arm}: {n} has no gradient in the plain model"
                continue
            sq += float(gp.double().square().sum())
            assert float(gt.abs().max()) > 0.0 or float(gp.abs().max()) == 0.0, f"{arm}: {n} region stayed zero"
            den = max(float(gp.double().norm()), 1e-4 * gmax)
            e = float((gt.double() - gp.double()).norm()) / den
            floor = float((grads_q[n].double() - gp.double()).norm()) / den
            tol = max(WHOLE_TOL[dtype], 3.0 * floor)
            assert e <= tol, f"{arm}: {n} relative error {e:.3g} > {tol:.3g} (plain model's own spread {floor:.3g})"
            if e > worst:
                worst, worst_name = e, n
            worst_ratio = max(worst_ratio, e / tol)
        REPORT[f"whole update {arm}[{mode}] worst parameter ({worst_name}) rel err"] = worst
        REPORT[f"whole update {arm}[{mode}] worst rel err / bound"] = worst_ratio
        print(f"\nwhole update {arm}[{mode}]: worst per-parameter relative error {worst:.3g} ({worst_name}); "
              f"gnorm_sq {gnorm_sq:.6g} vs plain {sq:.6g}")
        assert abs(gnorm_sq - sq) <= 1e-3 * sq, (arm, gnorm_sq, sq)
        if rec is not None:
            flat = (fp.grads.data_ptr(), fp.grads.data_ptr() + 4 * fp.numel)
            into_flat = [e for e in rec.ev if e["out"] is not None and flat[0] <= e["out"][0] < flat[1]]
            if dtype == torch.bfloat16:
                assert any(e["kind"] == "gemm" and e["acc"] == 2 and e["nb1"] > 1 and e["side"] for e in into_flat), \
                    "no split-K (S > 1) weight gradient on the side stream"
                assert any(e["kind"] == "colsum" and e["acc"] and e["out"][1] - e["out"][0] == 4 * 162 * 768
                           for e in into_flat), "the post-net group did not take the S-split + column sum"
            assert any(e["kind"] == "ln_bwd" for e in into_flat), "no bias gradient handed over to a LayerNorm"
    print(f"whole update [{mode}]: {time.time() - t0:.1f} s")


def RT_reset():
    from speecht5_b200.ops import RT
    RT.clear_static()
    RT.wgrad_stream = None
    RT._side_keep.clear()
    RT.probs_grad_heads = RT.probs_read_heads = 0
    RT.disable_device_seed()
    torch.cuda.synchronize()

"""Throughput mode against the reference model's own bf16 run (test infrastructure).

Three arms see one state dict and one batch:
  P  the product model in throughput mode (RT.dtype = bf16, fp32 master weights whose bf16 shadows the GEMMs read),
  T  the twin: the oracle (a plain-PyTorch restatement of the reference modules, with the reference's fp32 islands --
     softmax and GELU via .float(), the sinusoid tables) cast to bf16 on the same device: what the reference computes
     under fairseq's --bf16. Its criterion runs on its outputs cast to fp32, as the product's fp32 criterion kernels do,
  R  the same oracle in fp64. Its fp32 islands leave it a floor of ~1e-7 relative, far below bf16's 2^-8.

The weights and the float inputs are made bf16-representable before the arms are built (`bf16_exact`), so that P's bf16
shadows, T's bf16 parameters and R's fp64 parameters hold the same values and only the arithmetic differs.

For every compared quantity q, with e_X = ||X - R|| (X in {P, T}), the check is

    e_P(q) <= C * e_T(q) + F * ||R(q)||                                                             (1)

with C = 2 and F = 2^-12: throughput mode may be twice as far from fp64 as the reference's own bf16 run, plus a relative
floor well below one bf16 rounding. It is applied per utterance (L2 over the utterance's valid rows) and as a max-abs
version over the whole tensor, per scalar loss term and per parameter gradient. A gradient that is analytically zero
(R below F * gmax, e.g. k_proj.bias: softmax is invariant to a per-row shift) is held to ||P|| <= C ||T|| + F gmax.

A scalar is ONE draw of each arm's rounding error, not a norm over many elements that concentrates: for two independent
errors of equal spread, P(|e_P| > C |e_T|) = 1 - (2/pi) atan(C) (the ratio is Cauchy), 30 % at C = 2. So a scalar s =
sum_i a_i gets an a-priori floor instead of F |R|: U * sum_i |a_i| of R, U = 2^-8 the bf16 unit roundoff, i.e. what one
bf16 rounding of every term costs at most,

    e_P(s) <= C * e_T(s) + U * sum_i |a_i(R)|.                                                       (2)

Every loss term here is a mean or sum of non-negative terms (L1, L2, BCE, guided attention, label-smoothed CE, CTC), so
sum |a_i| = |R|. The gradient of a positional-encoding alpha is sum dy * pe over (utterance, frame, channel), a sum of
cancelling terms: `alpha_scales` records sum |dy * pe| from R's backward pass.

The largest e_P / (C e_T + F ||R||) of every check goes to REPORT; the test module prints it at the end."""
import torch

C_TWIN = 2.0
F_TWIN = 2.0 ** -12
U_BF16 = 2.0 ** -8
REPORT = {}  # check name -> largest e_P / bound seen


# ------------------------------------------------------------------------------------------------------ rounding
def bf16_exact(t):
    """A float tensor with every element rounded to the nearest bf16 value (same dtype); anything else unchanged."""
    if torch.is_tensor(t) and t.is_floating_point():
        return t.to(torch.bfloat16).to(t.dtype)
    return t


def cast_tree(obj, dtype=None, device=None):
    """Dicts / lists / tuples of tensors: float tensors to `dtype` (if given), every tensor to `device` (if given)."""
    if torch.is_tensor(obj):
        if dtype is not None and obj.is_floating_point():
            obj = obj.to(dtype)
        return obj.to(device) if device is not None else obj
    if isinstance(obj, dict):
        return {k: cast_tree(v, dtype, device) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(cast_tree(v, dtype, device) for v in obj)
    return obj


def round_tree(obj):
    """Every float tensor of a nested batch / state dict made bf16-representable."""
    if torch.is_tensor(obj):
        return bf16_exact(obj)
    if isinstance(obj, dict):
        return {k: round_tree(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(round_tree(v) for v in obj)
    return obj


def twin_and_reference(make, state, device):
    """T (bf16) and R (fp64) oracles built by `make()` from one (bf16-representable) state dict, on `device`."""
    arms = []
    for dtype in (torch.bfloat16, torch.float64):
        m = make()
        m.load_state_dict(state)
        arms.append(m.to(device=device, dtype=dtype))
    return arms


# ------------------------------------------------------------------------------------------------------ comparison
def _norm(x):
    return float(x.double().norm())


def ratio(p, t, r, C=C_TWIN, F=F_TWIN):
    """e_P / (C e_T + F ||R||) in the L2 norm; <= 1 passes (1)."""
    p, t, r = (x.detach().double() for x in (p, t, r))
    bound = C * _norm(t - r) + F * _norm(r)
    e = _norm(p - r)
    return e / bound if bound > 0 else (0.0 if e == 0 else float("inf"))


def ratio_max(p, t, r, C=C_TWIN, F=F_TWIN):
    """The max-abs version of (1) over the whole tensor."""
    p, t, r = (x.detach().double() for x in (p, t, r))
    bound = C * float((t - r).abs().max()) + F * float(r.abs().max())
    e = float((p - r).abs().max())
    return e / bound if bound > 0 else (0.0 if e == 0 else float("inf"))


def ratio_zero(p, t, gmax, C=C_TWIN, F=F_TWIN):
    """An analytically zero quantity: ||P|| <= C ||T|| + F gmax."""
    return _norm(p.detach()) / (C * _norm(t.detach()) + F * gmax)


class Twin:
    """Collects the checks of one case under a name prefix. `fails` lists every check whose ratio exceeds 1; `worst`
    is the largest ratio seen. With `report=False` nothing is recorded in REPORT (the sensitivity runs)."""

    def __init__(self, name, C=C_TWIN, F=F_TWIN, report=True):
        self.name, self.C, self.F, self.report = name, C, F, report
        self.fails, self.worst, self.worst_what, self.n = [], 0.0, None, 0

    def _record(self, what, q, group=None):
        self.n += 1
        if q > self.worst:
            self.worst, self.worst_what = q, what
        key = f"{self.name}: {group or what}"
        if self.report:
            REPORT[key] = max(q, REPORT.get(key, 0.0))
        if not q <= 1.0:
            self.fails.append((what, q))
        return q

    def tensor(self, what, p, t, r, rows=None, C=None):
        """Per utterance (leading axis; `rows[b]`: that utterance's valid extent along axis 1) and max-abs over all."""
        C = self.C if C is None else C
        worst = 0.0
        for b in range(r.shape[0]):
            n = None if rows is None else int(rows[b])
            sl = (lambda x: x[b]) if n is None else (lambda x: x[b, :n])
            worst = max(worst, self._record(f"{what}[{b}]", ratio(sl(p), sl(t), sl(r), C, self.F), f"{what} per utt"))
        if rows is None:
            pm, tm, rm = p, t, r
        else:
            keep = torch.arange(r.shape[1], device=r.device)[None, :] < torch.as_tensor(rows, device=r.device)[:, None]
            pm, tm, rm = p[keep], t[keep], r[keep]
        self._record(f"{what} max-abs", ratio_max(pm, tm, rm, C, self.F), f"{what} max-abs")
        return worst

    def scalar(self, what, p, t, r, abs_sum=None, group="loss terms"):
        """(2) for one scalar; abs_sum = sum |a_i| of R (default |R|: a mean or sum of non-negative terms)."""
        p, t, r = (float(x) for x in (p, t, r))
        abs_sum = abs(r) if abs_sum is None else float(abs_sum)
        bound = self.C * abs(t - r) + U_BF16 * abs_sum
        e = abs(p - r)
        return self._record(what, e / bound if bound > 0 else (0.0 if e == 0 else float("inf")), group)

    def grads(self, gp, gt, gr, C=None, scalar_abs=None):
        """Per parameter: gp / gt / gr map names to gradients (None: no gradient). Every parameter R differentiates
        must have a gradient in P and T. A one-element gradient is checked by (2) with scalar_abs[name] = sum |terms|."""
        scalar_abs = scalar_abs or {}
        C = self.C if C is None else C
        gmax = max(_norm(g) for g in gr.values() if g is not None)
        n = 0
        for name, r in gr.items():
            if r is None:
                continue
            p, t = gp.get(name), gt.get(name)
            if p is None or t is None:
                self.fails.append((f"grad {name} missing ({'P' if p is None else 'T'})", float("inf")))
                continue
            p, t = p.to(r.device), t.to(r.device)
            if _norm(r) <= self.F * gmax:
                self._record(f"grad {name} (zero)", ratio_zero(p, t, gmax, C, self.F), "grad analytically zero")
            elif r.numel() == 1:
                if name not in scalar_abs:
                    self.fails.append((f"grad {name}: a scalar without an a-priori scale", float("inf")))
                    continue
                self.scalar(f"grad {name}", p, t, r, scalar_abs[name], "grad scalar parameter")
            else:
                self._record(f"grad {name}", ratio(p, t, r, C, self.F), "grad per parameter")
            n += 1
        return n

    def verdict(self):
        return f"{self.name}: {self.n} checks, worst {self.worst:.3g} ({self.worst_what}); fails {self.fails[:6]}"

    def assert_ok(self):
        assert not self.fails, self.verdict()


def print_report():
    if REPORT:
        print(f"\nlargest e_P / (C e_T + F |R|) per check (C = {C_TWIN:g}, F = 2^{int(torch.log2(torch.tensor(F_TWIN)))}):")
        for k in sorted(REPORT):
            print(f"  {k:72s} {REPORT[k]:.3g}")


def alpha_scales(model):
    """Hooks every ScaledPositionalEncoding of an oracle: after a backward pass the returned dict maps
    '<module>.alpha' to sum |dy * pe| (the terms of that alpha's gradient), dy = the gradient of the module's output."""
    from oracle.speecht5_oracle import ScaledPositionalEncoding
    out = {}
    for name, m in model.named_modules():
        if isinstance(m, ScaledPositionalEncoding):
            def fwd(mod, inp, y, key=f"{name}.alpha"):
                pe = mod.table(y.size(1), mod.d_model, torch.float64).to(y.device)
                y.register_hook(lambda g: out.__setitem__(key, float((g.double() * pe).abs().sum())))
            m.register_forward_hook(fwd)
    return out


def param_grads(model, rename=None):
    """name -> gradient (detached copy; None where there is none) under the oracle's names."""
    rename = rename or {}
    return {rename.get(n, n): (p.grad.detach().clone() if p.grad is not None else None)
            for n, p in model.named_parameters()}

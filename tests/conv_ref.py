"""fp64 statements of the convolutions the host composes from st5_gemm_bf16 over overlapping-window operand views --
the post-net Conv1d k5 (ops.Conv1dK5Fn), the strided front-end layers 1-6 (frontend.StridedConvGeluFn), the grouped
positional conv (frontend.GroupedPosConvFn) and the HiFi-GAN convolutions (vocoder._conv_same, _conv_transpose) -- and
elementwise bounds for what the device returns. CPU or GPU (everything runs where its inputs live); no import of
speecht5_b200.

Statements: torch.nn.functional.conv1d / conv_transpose1d in float64 on exactly the values the GEMMs read.
  bf16 mode (RT.dtype = bfloat16): the bf16 activations as stored and bf16(w), the round-to-nearest shadow of the
    fp32 weight (st5_cast_bf16);
  parity mode (RT.dtype = float32): the fp32 activations and the fp32 weights; their split into bf16 parts is charged
    to the bound below;
  HiFi-GAN: the operand st5_lrelu_pad writes, bf16(fp32(x * slope)) for x < 0 (`lrelu_bf16`).
Gradients are the vector-Jacobian products of the same fp64 functions (`Conv.vjp`) with g = dy act'(pre), where pre
is the pre-activation the device saved (y.grad_fn.saved_tensors), so an error of the forward is not charged twice.
mag = the same function of |x|, |w| (and |g|): the sum of the absolute product terms of each output, elementwise.

Bounds, per element; u16 = 2^-8 and u32 = 2^-24 are the bf16 and fp32 unit roundoffs, K the contraction length of
the GEMM that produces the element:
  product, bf16 mode    C_ACC u32 sqrt(K) mag, the fp32-accumulation bound of the GEMM contract (C_ACC = 16,
                        tests/test_gemm_contract_gpu.py).
  product, parity mode  each operand v is split as hi = bf16(v), lo = bf16(v - hi), so |v - hi| <= u16 |v|,
                        r = v - hi - lo has |r| <= u16 |v - hi| <= u16^2 |v|, and |lo| <= u16 (1 + u16) |v|. The
                        three passes hi_x hi_w + hi_x lo_w + lo_x hi_w drop, per product term,
                          x w - (...) = lo_x lo_w + (hi_x + lo_x) r_w + r_x w,
                          |.| <= u16^2 [(1 + u16)^2 + (1 + u16^2) + 1] |x w| <= SPLIT |x w|,  SPLIT = 3.008 u16^2;
                        the passes accumulate in fp32 over magnitudes mag, u16 (1 + u16) mag and u16 (1 + u16) mag,
                        and the two accumulating passes round the running fp32 sum once more each (<= 1.01 u32 mag):
                          C_ACC u32 sqrt(K) (1 + 2 u16 (1 + u16)) mag + SPLIT mag + 3 u32 mag.
  epilogue              pre = acc + bias: + u32 |pre|; y = act(pre): |act'(pre)| e_pre + e_pre^2 + the evaluation
                        error of the device's activation (`act_eval`); + residual: + u32 |y|; the store: u_out |y|.
  gradients             g = dy act'(pre) as st5_act_bwd stores it (rowops_ref.act_bwd_bound, which includes the
                        rounding of g to its storage type, u16 |g| in bf16 mode); dx and dW add the product bound of
                        their GEMM over mag(|g|) and the propagated g error, vjp(e_g, |w|) / vjp(e_g, |x|). Sums the
                        host adds after the GEMMs (the strided layers' per-utterance dW, the post-net's split-K reduce
                        at the L2) add one u32 mag per term.

Margins. A dropped, duplicated or shifted tap, row or k-block changes an output by at least one product term, whose
typical size against mag is 1 / sqrt(K) (random signs). The bound at that element is about
(C_ACC u32 K + u_out) / sqrt(K) mag in bf16 mode (|ref| ~ mag / sqrt(K)), and in parity mode about
(C_ACC u32 K + SPLIT sqrt(K)) / sqrt(K) mag. One such term exceeds it by:
  post-net          K = 5 Cin   = 400 / 1280:  x 233 / x 195 (bf16), x 770 / x 349 (parity)
  strided, C = 512  K = k Cin   = 1024 - 2560: x 205 - x 158 (bf16), x 409 - x 210 (parity)
  positional conv   K = 128 cg  = 6144 / 8192: x 102 / x 85 (bf16), x 106 / x 84 (parity)
  weight gradients  K = frames, e.g. 2112 (post-net, B = 3, T = 700; fp32 output): x 496 (bf16), x 243 (parity)
  HiFi-GAN          K = k Cin   <= 11 x 512:   x 108 (bf16 only)
tests/test_conv_ref_cpu.py shows on the GEMM emulator that a dropped last k-block, a skipped split-K chunk, a phase
written one row off and a transposed-conv tap off by one each leave these bounds."""
import math

import torch
import torch.nn.functional as F

import rowops_ref as R

F64 = torch.float64
U32 = R.U32
U16 = R.U_BF16
TINY = R.TINY
C_EW = R.C_EW
C_ACC = 16.0
SPLIT = 3.008 * U16 * U16
A2 = 1.0  # |act''| <= 0.84 for both GELU forms, <= 0.77 for tanh: carries an error of pre into act(pre)


def unit(dtype):
    return U16 if dtype == torch.bfloat16 else U32


# ============================================================================================ statements
def conv1d_cl(x, w, *, stride=1, padding=0, dilation=1, groups=1, bias=None, length=None):
    """Conv1d on channels-last x [B, T, Cin] -> [B, T_out, Cout]; `length` keeps the first frames only (SamePad)."""
    y = F.conv1d(x.transpose(1, 2), w, bias, stride=stride, padding=padding, dilation=dilation, groups=groups)
    if length is not None:
        y = y[..., :length]
    return y.transpose(1, 2)


def conv_transpose1d_cl(x, w, *, stride, padding, bias=None):
    return F.conv_transpose1d(x.transpose(1, 2), w, bias, stride=stride, padding=padding).transpose(1, 2)


def weight_as_read(w, dtype):
    """The weight values the GEMM multiplies: bf16(w) in bf16 mode, w itself in parity mode."""
    return (w.to(torch.bfloat16) if dtype == torch.bfloat16 else w.float()).to(F64)


def lrelu_bf16(x, slope):
    """st5_lrelu_pad's output value: x for x > 0, else bf16(fp32(x * slope)) (slope 1: x)."""
    v = x.to(F64)
    neg = (v * R.f32(slope)).float().to(torch.bfloat16).to(F64)
    return torch.where(v > 0, v, neg)


class Conv:
    """fp64 y = fn(x, w) for a bilinear fn, its vector-Jacobian products and the magnitudes of all three."""

    def __init__(self, fn, x, w):
        self.fn, self.x, self.w = fn, x.to(F64), w.to(F64)

    def forward(self):
        return self.fn(self.x, self.w), self.fn(self.x.abs(), self.w.abs())

    def vjp(self, g, x=None, w=None):
        x = (self.x if x is None else x).detach().clone().requires_grad_()
        w = (self.w if w is None else w).detach().clone().requires_grad_()
        with torch.enable_grad():
            dx, dw = torch.autograd.grad(self.fn(x, w), (x, w), g.to(F64))
        return dx, dw

    def vjp_mag(self, gabs):
        """(|dx| terms, |dW| terms): the vjp of |g| through |x|, |w|."""
        return self.vjp(gabs, self.x.abs(), self.w.abs())


# ============================================================================================ bounds
def product_bound(mag, K, dtype):
    b = C_ACC * U32 * math.sqrt(K) * mag
    if dtype == torch.float32:
        b = b * (1 + 2 * U16 * (1 + U16)) + (SPLIT + 3 * U32) * mag
    return b


def act_ref(x, act):
    """The activation the device evaluates, in fp64: gelu (erf form, parity mode), gelu_tanh (the tanh form that
    ST5_ACT_GELU_TANH computes in bf16 mode), tanh, none."""
    if act == "gelu_tanh":
        return R.gelu_tanh(x)
    return R.act(x, act)


def act_eval(x, act):
    """|device act(x) - act_ref(x)| for an exact fp32 input x."""
    x = x.to(F64)
    y = act_ref(x, act)
    if act == "gelu":     # A&S erf through the approximate rcp / ex2 (rowops_ref.E_PHI)
        return x.abs() * R.E_PHI + C_EW * U32 * y.abs()
    if act == "gelu_tanh":  # 0.5 x (1 + t), t from tanh.approx: relative error of t <= 2^-10.98
        t = torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)).abs()
        return R.E_TANH_APPROX * 0.5 * x.abs() * t + C_EW * U32 * (y.abs() + 0.5 * x.abs())
    if act == "tanh":     # tanhf: 2 ulp
        return 4 * U32 * y.abs()
    assert act in (None, "none"), act
    return torch.zeros_like(y)


def epilogue(acc, e_acc, *, u_out, bias=None, act=None, residual=None):
    """Reference and bound of the GEMM epilogue over an accumulated product acc (bound e_acc):
    pre = acc + bias, y = act(pre) + residual, both stored in the output type (unit u_out)."""
    pre = acc if bias is None else acc + bias.to(F64)
    e_pre = e_acc + (U32 * pre.abs() if bias is not None else 0.0)
    if act in (None, "none"):
        y, e_y = pre, e_pre
    else:
        y = act_ref(pre, act)
        e_y = R.act_grad(pre, act).abs() * e_pre + A2 * e_pre * e_pre + act_eval(pre, act)
    if residual is not None:
        y = y + residual.to(F64)
        e_y = e_y + U32 * y.abs()
    return dict(pre=pre, e_pre=e_pre + u_out * pre.abs() + TINY, y=y, e_y=e_y + u_out * y.abs() + TINY)


def act_grad_input(dy, pre, act, u_g):
    """g = dy act'(pre) as st5_act_bwd stores it (type unit u_g), and its bound; act None: g = dy exactly."""
    if act in (None, "none"):
        g = dy.to(F64)
        return g, torch.zeros_like(g)
    return R.act_bwd_bound(dy, pre, act, u_g)


def grad_bounds(conv, g, e_g, *, K_dx, K_dw, dtype, u_dx, dx_extra=None, dw_sum_terms=0):
    """Reference and bounds of dx (stored in unit u_dx, + dx_extra fp32 added in the epilogue: the residual dy) and dW
    (fp32; dw_sum_terms fp32 additions of partial products after the GEMMs)."""
    dx, dw = conv.vjp(g)
    mdx, mdw = conv.vjp_mag(g.abs())
    pdx, pdw = conv.vjp(e_g, conv.x.abs(), conv.w.abs())
    e_dx = product_bound(mdx, K_dx, dtype) + pdx
    if dx_extra is not None:
        dx = dx + dx_extra.to(F64)
        e_dx = e_dx + U32 * dx.abs()
    e_dx = e_dx + u_dx * dx.abs() + TINY
    e_dw = product_bound(mdw, K_dw, dtype) + pdw + dw_sum_terms * U32 * mdw + TINY
    return dict(dx=dx, e_dx=e_dx, dw=dw, e_dw=e_dw)


def colsum_bound(g, e_g, rows_dims):
    """Bias gradient = column sums of g over `rows_dims` (st5_colsum, depth rowops_ref.C_COL) and its bound."""
    return g.sum(rows_dims), R.C_COL * U32 * g.abs().sum(rows_dims) + e_g.sum(rows_dims) + TINY


check = R.check

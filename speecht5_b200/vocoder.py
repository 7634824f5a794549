"""HiFi-GAN generator (mel -> waveform) on the device, inference only (SURVEY section 8a row 16; reference: the sibling
tree's SpeechUT/fairseq/fairseq/models/text_to_speech/hifigan.py:13-170 with the SpeechT5 vocoder configuration).

Every convolution is a window GEMM on the existing
wgmma kernel over channels-last activations (no im2col); the operand views are checked on the CPU through the GEMM
emulator against oracle/audio_oracle.py:HifiGanGenerator (tests/test_frontend_cpu.py).

* Conv1d(k, padding (k-1)/2): one batched GEMM over the zero-padded input, row t = the k*C contiguous elements from
  frame t, bias (and the residual of the ResBlock's second convolution, and the final tanh) in the epilogue.
* ConvTranspose1d(k = 2u, stride u, padding u/2): u phase GEMMs; phase r reads two neighbouring input frames and writes
  output frames r, r+u, ... (row pitch u*C_out).
* dilated Conv1d(dilation d): the leaky-ReLU that precedes it writes its result de-interleaved into d phase buffers
  (frame t -> phase t mod d); inside a phase the dilation is 1, and each phase GEMM writes its rows back with pitch d*C.
The leaky-ReLU, the zero padding and the de-interleave of every convolution input are ONE launch (st5_lrelu_pad); the
ResBlock averaging is a torch elementwise call."""
import torch
import torch.nn.functional as F

from . import kernels as K

LRELU_SLOPE = 0.1
HIFIGAN_CFG = dict(model_in_dim=80, upsample_initial_channel=512, upsample_rates=[4, 4, 4, 4],
                   upsample_kernel_sizes=[8, 8, 8, 8], resblock_kernel_sizes=[3, 7, 11],
                   resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]])


def _pad8(n):
    return (n + 7) // 8 * 8


def _bf16_rows(w2d):
    """fp32 [rows, cols] -> bf16 [rows, ld] with ld = cols rounded up to 8 (zero filled); returns (tensor, ld)."""
    rows, cols = w2d.shape
    ld = _pad8(cols)
    src = torch.zeros((rows, ld), dtype=torch.float32, device=w2d.device)
    src[:, :cols] = w2d
    out = torch.empty((rows, ld), dtype=torch.bfloat16, device=w2d.device)
    K.cast_bf16(src, out, None)
    return out, ld


class _Conv:
    """Conv1d weights [C_out, C_in, k] pre-arranged for the window GEMM: W2[co, j*C_in + ci]."""

    def __init__(self, weight, bias, dilation=1):
        self.cout, self.cin, self.k = weight.shape
        self.d = dilation
        self.w, self.ld = _bf16_rows(weight.permute(0, 2, 1).reshape(self.cout, self.k * self.cin).float())
        self.bias = bias.float().contiguous()


def _conv_same(x, conv, out=None, act=None, residual=None, pre_act_slope=None):
    """'same' Conv1d on channels-last x [B, T, C_in] (bf16) -> [B, T, C_out]. pre_act_slope: leaky-ReLU applied to the
    input while it is copied into the padded / de-interleaved operand buffer."""
    B, T, Cin = x.shape
    k, d, Cout = conv.k, conv.d, conv.cout
    x = x.contiguous()
    pad = (k * d - d) // 2
    y = out if out is not None else torch.empty((B, T, Cout), dtype=torch.bfloat16, device=x.device)
    for ph in range(d):
        # frames ph, ph+d, ... of the padded signal; output frame t = ph + d*m reads phase-frames m .. m+k-1
        n_out = (T - ph + d - 1) // d
        if n_out <= 0:
            continue
        n_in = n_out + k - 1
        # phase-frame i is padded index ph + d*i, i.e. x frame ph + d*i - pad: activation, zero borders and the
        # de-interleave in ONE launch (st5_lrelu_pad; slope 1 = plain copy)
        buf = torch.empty((B, n_in, Cin), dtype=torch.bfloat16, device=x.device)
        K.lrelu_pad(x, buf, d, ph, pad, pre_act_slope if pre_act_slope is not None else 1.0)
        kw = dict(M=n_out, N=Cout, K=k * Cin, a_ld=Cin, b_ld=conv.ld, c_ld=d * Cout, nb1=B, nb2=1, a_bs=(n_in * Cin, 0),
                  b_bs=(0, 0), c_bs=(T * Cout, 0), bias=conv.bias, act=act)
        if residual is not None:
            kw["residual"] = residual.reshape(-1)[ph * Cout:]
        K.gemm(buf, conv.w, y.reshape(-1)[ph * Cout:], **kw)
    return y


class _ConvT:
    """ConvTranspose1d weights [C_in, C_out, k], stride u, padding p, split into u phases of `taps` input frames."""

    def __init__(self, weight, bias, stride, padding):
        self.cin, self.cout, self.k = weight.shape
        self.u, self.p = stride, padding
        self.taps = (self.k + stride - 1) // stride
        self.bias = bias.float().contiguous()
        self.phases = []
        for r in range(stride):
            ds = [dd for dd in range(-(self.taps - 1), self.taps) if 0 <= r + padding - stride * dd < self.k]
            # output n = u*m + r  <-  sum_dd x[m + dd] . W[:, :, r + p - u*dd]; window order: dd ascending
            wr = torch.stack([weight[:, :, r + padding - stride * dd] for dd in ds], dim=0)  # [taps, C_in, C_out]
            w2 = wr.permute(2, 0, 1).reshape(self.cout, len(ds) * self.cin).float()
            w, ld = _bf16_rows(w2)
            self.phases.append((min(ds), len(ds), w, ld))


def _conv_transpose(x, ct, pre_act_slope=None):
    B, T, Cin = x.shape
    fr = ct.taps - 1
    buf = torch.empty((B, T + 2 * fr, Cin), dtype=torch.bfloat16, device=x.device)
    K.lrelu_pad(x.contiguous(), buf, 1, 0, fr, pre_act_slope if pre_act_slope is not None else 1.0)
    y = torch.empty((B, T * ct.u, ct.cout), dtype=torch.bfloat16, device=x.device)
    Tp = T + 2 * fr
    for r, (d0, nt, w, ld) in enumerate(ct.phases):
        a = buf.reshape(-1)[(fr + d0) * Cin:]
        K.gemm(a, w, y.reshape(-1)[r * ct.cout:], M=T, N=ct.cout, K=nt * Cin, a_ld=Cin, b_ld=ld, c_ld=ct.u * ct.cout,
               nb1=B, nb2=1, a_bs=(Tp * Cin, 0), b_bs=(0, 0), c_bs=(T * ct.u * ct.cout, 0), bias=ct.bias)
    return y


class HifiGanGenerator:
    """Inference-only generator built from a state dict with the oracle's / reference's key names (weight norm folded:
    `conv_pre.weight`, `ups.{i}.weight`, `resblocks.{r}.convs1.{j}.weight`, ..., `conv_post.weight`, `mean`, `scale`)."""

    def __init__(self, state_dict, cfg=None, device="cuda"):
        cfg = dict(HIFIGAN_CFG, **(cfg or {}))
        self.cfg = cfg
        sd = {k: v.to(device) for k, v in state_dict.items()}
        self.mean, self.scale = sd["mean"].float(), sd["scale"].float()
        self.conv_pre = _Conv(sd["conv_pre.weight"], sd["conv_pre.bias"])
        self.ups = [_ConvT(sd[f"ups.{i}.weight"], sd[f"ups.{i}.bias"], u, (k - u) // 2)
                    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"]))]
        self.num_kernels = len(cfg["resblock_kernel_sizes"])
        self.resblocks = []
        r = 0
        for _ in cfg["upsample_rates"]:
            for _k, dil in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]):
                c1 = [_Conv(sd[f"resblocks.{r}.convs1.{j}.weight"], sd[f"resblocks.{r}.convs1.{j}.bias"], d)
                      for j, d in enumerate(dil)]
                c2 = [_Conv(sd[f"resblocks.{r}.convs2.{j}.weight"], sd[f"resblocks.{r}.convs2.{j}.bias"], 1)
                      for j, _d in enumerate(dil)]
                self.resblocks.append((c1, c2))
                r += 1
        self.conv_post = _Conv(sd["conv_post.weight"], sd["conv_post.bias"])

    @torch.no_grad()
    def __call__(self, spectrogram, normalize_before=True):
        """spectrogram [B, T, 80] fp32 log-mel -> waveform [B, T * prod(upsample_rates)] fp32."""
        K._require_cuda(spectrogram)
        x = spectrogram.float()
        if normalize_before:
            x = (x - self.mean) / self.scale
        B, T, C0 = x.shape
        ld0 = _pad8(C0)
        xb = torch.zeros((B, T, ld0), dtype=torch.bfloat16, device=x.device)
        xb[..., :C0] = x.to(torch.bfloat16)
        if ld0 != C0:
            raise NotImplementedError("model_in_dim must be a multiple of 8 (80 in the release)")
        x = _conv_same(xb, self.conv_pre)
        for i, up in enumerate(self.ups):
            x = _conv_transpose(x, up, pre_act_slope=LRELU_SLOPE)
            xs = None
            for j in range(self.num_kernels):
                c1s, c2s = self.resblocks[i * self.num_kernels + j]
                h = x
                for c1, c2 in zip(c1s, c2s):
                    t = _conv_same(h, c1, pre_act_slope=LRELU_SLOPE)
                    h = _conv_same(t, c2, residual=h, pre_act_slope=LRELU_SLOPE)
                xs = h.float() if xs is None else xs + h.float()
            x = (xs / self.num_kernels).to(torch.bfloat16)
        y = torch.empty((x.shape[0], x.shape[1], 1), dtype=torch.float32, device=x.device)
        _conv_same(x, self.conv_post, out=y, act="tanh", pre_act_slope=0.01)  # (default slope here, reference :165)
        return y[..., 0]

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
ResBlock averaging is a torch elementwise call.

Ragged batches (`HifiGanGenerator.vocode`): the utterances are padded to one length and every operand staging takes the
utterance's length at the current resolution (st5_lrelu_pad_len), so each convolution reads zeros past an utterance's
end exactly as it does when the utterance is vocoded alone; every other step is row-independent (the GEMM rows, the
epilogue, the elementwise calls). The whole pass is one captured CUDA graph per (batch, length bucket)."""
import math

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


def _stage(x, buf, d, ph, pad, slope, lengths, len_mult):
    if lengths is None:
        K.lrelu_pad(x, buf, d, ph, pad, slope)
    else:
        K.lrelu_pad_len(x, buf, d, ph, pad, slope, lengths, len_mult)


def _conv_same(x, conv, out=None, act=None, residual=None, pre_act_slope=None, lengths=None, len_mult=1):
    """'same' Conv1d on channels-last x [B, T, C_in] (bf16) -> [B, T, C_out]. pre_act_slope: leaky-ReLU applied to the
    input while it is copied into the padded / de-interleaved operand buffer. lengths (int32 [B] device tensor, times
    len_mult = frames of x): frames of row b at or past its length are read as zeros, as if x ended there; the output
    rows past it are then not meaningful."""
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
        _stage(x, buf, d, ph, pad, pre_act_slope if pre_act_slope is not None else 1.0, lengths, len_mult)
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


def _conv_transpose(x, ct, pre_act_slope=None, lengths=None, len_mult=1):
    B, T, Cin = x.shape
    fr = ct.taps - 1
    buf = torch.empty((B, T + 2 * fr, Cin), dtype=torch.bfloat16, device=x.device)
    _stage(x.contiguous(), buf, 1, 0, fr, pre_act_slope if pre_act_slope is not None else 1.0, lengths, len_mult)
    y = torch.empty((B, T * ct.u, ct.cout), dtype=torch.bfloat16, device=x.device)
    Tp = T + 2 * fr
    for r, (d0, nt, w, ld) in enumerate(ct.phases):
        a = buf.reshape(-1)[(fr + d0) * Cin:]
        K.gemm(a, w, y.reshape(-1)[r * ct.cout:], M=T, N=ct.cout, K=nt * Cin, a_ld=Cin, b_ld=ld, c_ld=ct.u * ct.cout,
               nb1=B, nb2=1, a_bs=(Tp * Cin, 0), b_bs=(0, 0), c_bs=(T * ct.u * ct.cout, 0), bias=ct.bias)
    return y


def _fold(g, v):
    """torch.nn.utils.weight_norm(dim=0): weight = v * (g / ||v||), the norm over every dimension but the first."""
    norm = v.reshape(v.size(0), -1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))
    return v * (g / norm)


def plain_state_dict(state_dict):
    """A generator state dict in the key names this module reads (`conv_pre`, `ups.{i}`, `resblocks.{r}.convs1.{j}`,
    `conv_post`, `mean`, `scale`, plain `.weight` / `.bias`), from any of the names the same tensors are published under:
    fairseq / SpeechUT (`ups.{i}`), HuggingFace SpeechT5HifiGan (`upsampler.{i}`), with weight norm either folded or as
    `weight_g` / `weight_v` pairs."""
    out = {}
    for k, v in state_dict.items():
        if k.endswith(".weight_v"):
            continue
        if k.endswith(".weight_g"):
            base = k[:-len("_g")]
            k, v = base, _fold(v, state_dict[base + "_v"])
        if k.startswith("upsampler."):
            k = "ups." + k[len("upsampler."):]
        out[k] = v
    return out


class HifiGanGenerator:
    """Inference-only generator built from a state dict (key names: see plain_state_dict; a state dict without `mean` /
    `scale` normalises with 0 / 1). cfg: the fields of HIFIGAN_CFG, named as in SpeechT5HifiGanConfig, plus
    `leaky_relu_slope`; other keys are ignored, so a HuggingFace config.json dict can be passed as it is."""

    def __init__(self, state_dict, cfg=None, device="cuda"):
        cfg = dict(cfg or {})
        self.lrelu_slope = float(cfg.get("leaky_relu_slope", LRELU_SLOPE))
        cfg = dict(HIFIGAN_CFG, **{k: v for k, v in cfg.items() if k in HIFIGAN_CFG})
        self.cfg = cfg
        sd = {k: v.to(device) for k, v in plain_state_dict(state_dict).items()}
        C0 = cfg["model_in_dim"]
        self.mean = sd["mean"].float() if "mean" in sd else torch.zeros(C0, device=device)
        self.scale = sd["scale"].float() if "scale" in sd else torch.ones(C0, device=device)
        self.device = self.mean.device
        self.hop = math.prod(cfg["upsample_rates"])  # waveform samples per mel frame
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
        self._graphs = {}  # (B, T_bucket, normalize_before, device) -> _VocodeGraph

    @torch.no_grad()
    def __call__(self, spectrogram, normalize_before=True):
        """spectrogram [B, T, 80] fp32 log-mel -> waveform [B, T * prod(upsample_rates)] fp32."""
        K._require_cuda(spectrogram)
        return self._forward(spectrogram, normalize_before)

    def _forward(self, spectrogram, normalize_before, lengths=None):
        """The generator on [B, T, model_in_dim]; lengths (int32 [B] device tensor, mel frames): row b is computed as
        if the input ended at its length (output samples past lengths[b] * prod(upsample_rates) are not meaningful)."""
        x = spectrogram.float()
        if normalize_before:
            x = (x - self.mean) / self.scale
        B, T, C0 = x.shape
        ld0 = _pad8(C0)
        xb = torch.zeros((B, T, ld0), dtype=torch.bfloat16, device=x.device)
        xb[..., :C0] = x.to(torch.bfloat16)
        if ld0 != C0:
            raise NotImplementedError("model_in_dim must be a multiple of 8 (80 in the release)")
        x = _conv_same(xb, self.conv_pre, lengths=lengths)
        mult = 1  # frames of x per mel frame
        for i, up in enumerate(self.ups):
            x = _conv_transpose(x, up, pre_act_slope=self.lrelu_slope, lengths=lengths, len_mult=mult)
            mult *= up.u
            xs = None
            for j in range(self.num_kernels):
                c1s, c2s = self.resblocks[i * self.num_kernels + j]
                h = x
                for c1, c2 in zip(c1s, c2s):
                    t = _conv_same(h, c1, pre_act_slope=self.lrelu_slope, lengths=lengths, len_mult=mult)
                    h = _conv_same(t, c2, residual=h, pre_act_slope=self.lrelu_slope, lengths=lengths, len_mult=mult)
                xs = h.float() if xs is None else xs + h.float()
            x = (xs / self.num_kernels).to(torch.bfloat16)
        y = torch.empty((x.shape[0], x.shape[1], 1), dtype=torch.float32, device=x.device)
        # (default slope here, reference :165)
        _conv_same(x, self.conv_post, out=y, act="tanh", pre_act_slope=0.01, lengths=lengths, len_mult=mult)
        return y[..., 0]

    def _check_mels(self, mels):
        """Host-side validation of vocode's input (raises ValueError; nothing is launched)."""
        if not isinstance(mels, (list, tuple)) or len(mels) == 0:
            raise ValueError("vocode takes a non-empty list of [L, model_in_dim] mel tensors")
        C0 = self.cfg["model_in_dim"]
        for b, m in enumerate(mels):
            if not torch.is_tensor(m) or m.dim() != 2 or m.shape[1] != C0:
                raise ValueError(f"mel {b}: expected a [L, {C0}] tensor, got "
                                 f"{tuple(m.shape) if torch.is_tensor(m) else type(m).__name__}")
            if m.shape[0] < 1:
                raise ValueError(f"mel {b}: empty (L = 0)")
            if m.dtype != torch.float32:
                raise ValueError(f"mel {b}: dtype {m.dtype}, expected torch.float32")
            if m.device != self.device:
                raise ValueError(f"mel {b}: on {m.device}, the vocoder is on {self.device}")

    @torch.no_grad()
    def vocode(self, mels, normalize_before=True):
        """Vocode utterances of different lengths in one CUDA-graph replay: mels = list of [L_b, model_in_dim] fp32
        device tensors -> list of [L_b * prod(upsample_rates)] fp32 waveforms, each bitwise equal to
        self(mels[b][None], normalize_before)[0]. The batch is padded to a bucket of 64 frames; one graph is captured
        per (B, bucket, normalize_before, device) and kept on the generator."""
        self._check_mels(mels)
        T_b = max(64, (max(m.shape[0] for m in mels) + 63) // 64 * 64)
        key = (len(mels), T_b, bool(normalize_before), str(self.device))
        vg = self._graphs.get(key)
        if vg is None:
            vg = self._graphs[key] = _VocodeGraph(self, len(mels), T_b, bool(normalize_before))
        return vg.run(mels)


class _VocodeGraph:
    """One generator pass over B utterances padded to T_bucket frames, reading the static buffers `mel` [B, T_bucket,
    model_in_dim] and `lengths` (int32 [B]): captured once, replayed for every batch of the same size and bucket. Frames
    of `mel` past an utterance's length are never read. capture=False runs the same body eagerly."""

    def __init__(self, gen, B, T_bucket, normalize_before, capture=True):
        self.gen, self.B, self.T, self.normalize_before, self.capture = gen, B, T_bucket, normalize_before, capture
        dev = gen.device
        self.mel = torch.zeros((B, T_bucket, gen.cfg["model_in_dim"]), dtype=torch.float32, device=dev)
        self.lengths = torch.zeros(B, dtype=torch.int32, device=dev)
        self.graph, self.out, self.launches = None, None, 0

    def _body(self):
        n0 = K.LAUNCHES
        out = self.gen._forward(self.mel, self.normalize_before, self.lengths)
        self.launches = K.LAUNCHES - n0  # library kernels per pass (a replay does not go through kernels.py)
        return out

    def _capture(self):
        dev = self.gen.device
        stream = torch.cuda.Stream(device=dev)
        stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(stream):
            self._body()  # warm-up outside the capture (first-call setup of the library and the allocator)
            stream.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                self.out = self._body()
        torch.cuda.current_stream(dev).wait_stream(stream)
        self.graph = g

    def run(self, mels):
        lens = [m.shape[0] for m in mels]
        assert len(mels) == self.B and max(lens) <= self.T
        for b, m in enumerate(mels):
            self.mel[b, :lens[b]].copy_(m)
        self.lengths.copy_(torch.tensor(lens, dtype=torch.int32))
        if not self.capture:
            self.out = self._body()
        else:
            if self.graph is None:
                self._capture()
            self.graph.replay()
        hop = self.gen.hop
        return [self.out[b, :L * hop].clone() for b, L in enumerate(lens)]

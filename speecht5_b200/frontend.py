"""Waveform feature extractor of the speech-input branch (SURVEY section 8a row 2; reference
speecht5/models/modules/speech_encoder_prenet.py:277-374): seven bias-free Conv1d layers
[(512,10,5)] + [(512,3,2)]*4 + [(512,2,2)]*2 with GELU after each; mode "default" (Base recipes) puts a GroupNorm(512
groups) after the first, mode "layer_norm" (t5_transformer_large, models/speecht5.py:1421) a LayerNorm over the channels
of every frame after every conv (:308-318).

The index algebra is checked on the CPU against torch's convolutions through a GEMM emulator
(tests/test_frontend_cpu.py), the device path against the oracle and the reference fixtures (tests/test_frontend_gpu.py,
tests/test_ref_pin_gpu.py). The TTS path does not import this module.

Device formulation (channels-last activations [B, T, C] throughout, no im2col, no transposes):
* layer 0: csrc/conv_frontend.cu -- conv + GroupNorm + GELU fused, the convolution recomputed from the waveform in
  every pass (kernels.conv0_gn_gelu_fwd / _bwd); in "layer_norm" mode conv + per-frame LayerNorm + GELU in ONE pass, a
  warp per frame (kernels.conv0_ln_gelu_fwd / _bwd);
* layers 1..6 in "layer_norm" mode: the same window GEMM without an epilogue activation, the row LayerNorm kernel of
  the transformer blocks (ops.residual_layer_norm, fp32 statistics) and a stand-alone GELU (kernels.act_fwd / act_bwd);
* layers 1..6 forward: ONE batched wgmma GEMM each over an overlapping-window view of the input -- row t of
  utterance b is the k*C_in contiguous elements starting at frame t*stride (row pitch stride*C_in) -- with GELU and
  the pre-activation store in the epilogue;
* input gradient: the transposed convolution split by output phase r = i mod stride; phase r is a window GEMM over
  the (front-padded) gradient with the taps t = r, r+stride, ... in reverse order, written with row pitch stride*C_in;
* weight gradient: per utterance dW2[b] = g_b^T . windows_b (both operands read MN-major), summed over b."""
import numpy as np
import torch

from . import kernels as K
from .ops import RT, _resolve_act, _split


def _passes(a, b, out, kw, epi=None):
    """One GEMM in bf16 mode; hi*hi + hi*lo + lo*hi (fp32 accumulate in `out`) in parity mode. a, b: (hi, lo) pairs."""
    a_hi, a_lo = a
    b_hi, b_lo = b
    epi = epi or {}
    if a_lo is None and b_lo is None:
        return K.gemm(a_hi, b_hi, out, **kw, **epi)
    assert out.dtype == torch.float32
    K.gemm(a_hi, b_hi, out, **kw)
    K.gemm(a_hi, b_lo, out, accumulate=True, **kw)
    K.gemm(a_lo, b_hi, out, accumulate=True, **kw, **epi)
    return out


def _off(pair, elems):
    """The (hi, lo) operand pair advanced by `elems` elements of the flat buffer."""
    return tuple(None if t is None else t.reshape(-1)[elems:] for t in pair)


def conv_out_len(T, k, s):
    return (T - k) // s + 1


class StridedConvGeluFn(torch.autograd.Function):
    """y = GELU(Conv1d(C_in -> C_out, k, stride, no bias)(x)) on channels-last x [B, T, C_in] -> [B, T_out, C_out];
    activation=None leaves the convolution alone (the "layer_norm" extractor normalises before its GELU)."""

    @staticmethod
    def forward(ctx, x, weight, stride, activation="gelu"):
        x = x.contiguous()
        B, T, Cin = x.shape
        Cout, _, k = weight.shape
        s = int(stride)
        To = conv_out_len(T, k, s)
        act = _resolve_act(activation, x.dtype)
        w2 = RT.shadow(("fe_f", id(weight)), lambda: weight.detach().permute(0, 2, 1).reshape(Cout, k * Cin))
        xa = _split(x.view(B * T, Cin))
        y = torch.empty((B, To, Cout), dtype=x.dtype, device=x.device)
        pre = torch.empty_like(y) if act is not None else None
        kw = dict(M=To, N=Cout, K=k * Cin, a_ld=s * Cin, b_ld=k * Cin, c_ld=Cout, nb1=B, nb2=1, a_bs=(T * Cin, 0),
                  b_bs=(0, 0), c_bs=(To * Cout, 0))
        _passes(xa, w2, y, kw, dict(act=act, c_pre=pre) if act is not None else None)
        ctx.save_for_backward(weight, pre)
        ctx.xa = xa
        ctx.meta = (B, T, Cin, Cout, k, s, To, act)
        return y

    @staticmethod
    def backward(ctx, dy):
        weight, pre = ctx.saved_tensors
        B, T, Cin, Cout, k, s, To, act = ctx.meta
        dev, dt = dy.device, dy.dtype
        jmax = (k + s - 1) // s                      # taps per output phase, at most
        mmax = (T + s - 1) // s                      # rows of one phase of dx, at most
        front = jmax - 1
        rows_p = front + max(To, mmax) + jmax        # zero rows in front (window history) and behind (untouched tail)
        gp = torch.zeros((B, rows_p, Cout), dtype=dt, device=dev)
        g = gp[:, front:front + To]
        # g = dy * gelu'(pre), written straight into the padded buffer the phase GEMMs read
        if act is not None:
            gtmp = torch.empty((B, To, Cout), dtype=dt, device=dev)
            K.act_bwd(dy.contiguous(), pre, gtmp, act)
            g.copy_(gtmp)
        else:
            g.copy_(dy)
        ga = _split(gp.view(B * rows_p, Cout))
        # ---- input gradient, one window GEMM per phase r: dx[b, s*m + r, :] = sum_q gpad[b, m + q', :] . Wr[q]
        dx = torch.empty((B, T, Cin), dtype=dt, device=dev)  # every frame belongs to exactly one phase
        for r in range(s):
            taps = list(range(r, k, s))              # t = r + s*j, j = 0..J-1
            J = len(taps)
            Mr = (T - r + s - 1) // s                # x frames with index = r (mod s)
            if Mr <= 0:
                continue
            if J == 0:
                dx[:, r::s].zero_()
                continue
            # window position q <-> tap j = J-1-q; W_r[ci, q*Cout + co] = W[co, ci, r + s*(J-1-q)]
            # (slice + flip, not a Python index list: that would be a host tensor copied to the device -- illegal under
            #  CUDA-graph capture -- every time the shadow is rebuilt after an optimizer step)
            wr = RT.shadow(("fe_b", id(weight), r), lambda r=r, J=J: weight.detach()[:, :, r::s].flip(2)
                           .permute(1, 2, 0).reshape(Cin, J * Cout))
            a_ops = _off(ga, (front - (J - 1)) * Cout)
            out_r = dx.reshape(-1)[r * Cin:]
            kw = dict(M=Mr, N=Cin, K=J * Cout, a_ld=Cout, b_ld=J * Cout, c_ld=s * Cin, nb1=B, nb2=1,
                      a_bs=(rows_p * Cout, 0), b_bs=(0, 0), c_bs=(T * Cin, 0))
            _passes(a_ops, wr, out_r, kw)
        # ---- weight gradient: dW2[b][co, t*Cin + ci] = sum_o g[b, o, co] * x[b, s*o + t, ci]
        dW2 = torch.empty((B, Cout, k * Cin), dtype=torch.float32, device=dev)
        kw = dict(M=Cout, N=k * Cin, K=To, a_mn=True, b_mn=True, a_ld=Cout, b_ld=s * Cin, c_ld=k * Cin, nb1=B, nb2=1,
                  a_bs=(rows_p * Cout, 0), b_bs=(T * Cin, 0), c_bs=(Cout * k * Cin, 0))
        _passes(_off(ga, front * Cout), ctx.xa, dW2, kw)
        dW = dW2.sum(0).view(Cout, k, Cin).permute(0, 2, 1).contiguous()
        ctx.xa = None
        return dx, dW, None, None


class GeluFn(torch.autograd.Function):
    """Stand-alone GELU (exact erf form in parity mode, tanh form on bf16 activations) behind the per-frame LayerNorm."""

    @staticmethod
    def forward(ctx, z):
        z = z.contiguous()
        act = _resolve_act("gelu", z.dtype)
        y = torch.empty_like(z)
        K.act_fwd(z, y, act)
        ctx.save_for_backward(z)
        ctx.act = act
        return y

    @staticmethod
    def backward(ctx, dy):
        (z,) = ctx.saved_tensors
        dz = torch.empty_like(z)
        K.act_bwd(dy.contiguous(), z, dz, ctx.act)
        return dz


class Conv0LayerNormGeluFn(torch.autograd.Function):
    """Layer 0 of the "layer_norm" extractor: waveform [B, n] fp32 -> GELU(LayerNorm_C(Conv1d(1 -> C, k, stride)))
    channels-last [B, T0, C]; per-frame statistics (fp32) saved for the backward."""

    @staticmethod
    def forward(ctx, wave, weight, gamma, beta, stride, eps, out_dtype):
        wave = wave.float().contiguous()
        B, n = wave.shape
        Cc, _, k = weight.shape
        s = int(stride)
        T0 = conv_out_len(n, k, s)
        act = _resolve_act("gelu", out_dtype)
        w2 = weight.detach().reshape(Cc, k).float().contiguous()
        y = torch.empty((B, T0, Cc), dtype=out_dtype, device=wave.device)
        mean = torch.empty((B * T0,), dtype=torch.float32, device=wave.device)
        rstd = torch.empty_like(mean)
        K.conv0_ln_gelu_fwd(wave, w2, gamma.detach().float(), beta.detach().float(), y, mean, rstd, s, eps, act)
        ctx.save_for_backward(wave, w2, gamma, beta, mean, rstd)
        ctx.meta = (s, act, tuple(weight.shape))
        return y

    @staticmethod
    def backward(ctx, dy):
        wave, w2, gamma, beta, mean, rstd = ctx.saved_tensors
        s, act, wshape = ctx.meta
        dw = torch.zeros_like(w2)
        dg = torch.zeros(w2.shape[0], dtype=torch.float32, device=w2.device)
        db = torch.zeros_like(dg)
        K.conv0_ln_gelu_bwd(dy.contiguous(), wave, w2, gamma.detach().float(), beta.detach().float(), mean, rstd, dw, dg,
                            db, s, act)
        return None, dw.view(wshape), dg, db, None, None, None


class Conv0GroupNormGeluFn(torch.autograd.Function):
    """Layer 0: waveform [B, n] fp32 -> GELU(GroupNorm_C(Conv1d(1 -> C, k, stride))) channels-last [B, T0, C]."""

    @staticmethod
    def forward(ctx, wave, weight, gamma, beta, stride, eps, out_dtype):
        wave = wave.float().contiguous()
        B, n = wave.shape
        Cc, _, k = weight.shape
        s = int(stride)
        T0 = conv_out_len(n, k, s)
        act = _resolve_act("gelu", out_dtype)
        w2 = weight.detach().reshape(Cc, k).float().contiguous()
        y = torch.empty((B, T0, Cc), dtype=out_dtype, device=wave.device)
        mean = torch.empty((B, Cc), dtype=torch.float32, device=wave.device)
        rstd = torch.empty_like(mean)
        K.conv0_gn_gelu_fwd(wave, w2, gamma.detach().float(), beta.detach().float(), y, mean, rstd, s, eps, act)
        ctx.save_for_backward(wave, w2, gamma, beta, mean, rstd)
        ctx.meta = (s, act, tuple(weight.shape))
        return y

    @staticmethod
    def backward(ctx, dy):
        wave, w2, gamma, beta, mean, rstd = ctx.saved_tensors
        s, act, wshape = ctx.meta
        dw = torch.zeros_like(w2)
        dg = torch.zeros_like(mean[0])
        db = torch.zeros_like(mean[0])
        K.conv0_gn_gelu_bwd(dy.contiguous(), wave, w2, gamma.detach().float(), beta.detach().float(), mean, rstd, dw, dg,
                            db, s, act)
        return None, dw.view(wshape), dg, db, None, None, None


CONV_FEATURE_LAYERS = [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2


class ConvFeatureExtractor(torch.nn.Module):
    """speech_encoder_prenet.py:277-374, modes "default" (the Base recipes) and "layer_norm" (t5_transformer_large).
    Parameter names follow the reference: `conv_layers.{i}.0.weight` [C_out, C_in, k]; GroupNorm affine at
    `conv_layers.0.2.{weight,bias}`; in "layer_norm" mode the norm of block i sits between two TransposeLast modules,
    `conv_layers.{i}.2.1.{weight,bias}` (:308-318). Output is channels-last [B, T, C] -- the reference's [B, C, T]
    transposed, which is what its caller does next (:169)."""

    def __init__(self, conv_layers=None, mode="default", conv_bias=False):
        super().__init__()
        if mode not in ("default", "layer_norm") or conv_bias:
            raise NotImplementedError("extractor_mode default / layer_norm without conv bias (the reference's recipes) are built")
        self.mode = mode
        self.specs = list(conv_layers or CONV_FEATURE_LAYERS)
        assert self.specs[0][1] <= 16
        self.conv_layers = torch.nn.ModuleList()
        in_d = 1
        for i, (dim, k, s) in enumerate(self.specs):
            conv = torch.nn.Conv1d(in_d, dim, k, stride=s, bias=False)
            torch.nn.init.kaiming_normal_(conv.weight)
            mods = [conv, torch.nn.Dropout(0.0)]
            if mode == "layer_norm":  # Sequential(TransposeLast, Fp32LayerNorm, TransposeLast): the key layout only
                mods.append(torch.nn.Sequential(torch.nn.Identity(), torch.nn.LayerNorm(dim), torch.nn.Identity()))
            elif i == 0:
                mods.append(torch.nn.GroupNorm(dim, dim, affine=True))
            mods.append(torch.nn.GELU())
            self.conv_layers.append(torch.nn.Sequential(*mods))
            in_d = dim

    def forward(self, wave):
        if not wave.is_cuda:
            raise RuntimeError("speecht5_b200 kernels need CUDA tensors (no CPU fallback)")
        return self._layers(wave)

    def _layers(self, wave):
        blk0 = self.conv_layers[0]
        if self.mode == "layer_norm":
            from . import ops
            ln0 = blk0[2][1]
            x = Conv0LayerNormGeluFn.apply(wave, blk0[0].weight, ln0.weight, ln0.bias, self.specs[0][2], ln0.eps, RT.dtype)
            for i in range(1, len(self.specs)):
                blk = self.conv_layers[i]
                u = StridedConvGeluFn.apply(x, blk[0].weight, self.specs[i][2], None)
                x = GeluFn.apply(ops.residual_layer_norm(u, None, blk[2][1]))
            return x
        x = Conv0GroupNormGeluFn.apply(wave, blk0[0].weight, blk0[2].weight, blk0[2].bias, self.specs[0][2],
                                       blk0[2].eps, RT.dtype)
        for i in range(1, len(self.specs)):
            x = StridedConvGeluFn.apply(x, self.conv_layers[i][0].weight, self.specs[i][2])
        return x

    def get_out_seq_lens_tensor(self, lengths):
        out = lengths.clone()
        for _, k, s in self.specs:
            out = torch.div(out - k, s, rounding_mode="floor") + 1
        return out


def _cast_pair(w2d):
    """(hi, lo) bf16 operands of a freshly computed fp32 2-D tensor (not a Parameter: nothing to cache on)."""
    w2d = w2d.detach().float().contiguous()
    hi = torch.empty(w2d.shape, dtype=torch.bfloat16, device=w2d.device)
    lo = torch.empty_like(hi) if RT.dtype == torch.float32 else None
    K.cast_bf16(w2d, hi, lo)
    return hi, lo


class GroupedPosConvFn(torch.autograd.Function):
    """y = x + GELU(SamePad(Conv1d(C, C, k, padding k//2, groups G)(x)) + bias) on channels-last x [B, T, C]
    (speech_encoder_prenet.py:105-119,187-192; k even: the last output frame is dropped). `weight` [C, C/G, k] is the
    weight-normed tensor g*v/||v|| computed by the caller with torch ops, so its gradient flows on to g and v.

    Per group: the input is regrouped once into a zero-padded group-major buffer [G, B, T+k, C/G]; the convolution is
    then a window GEMM (row t = the k*(C/G) contiguous elements from frame t, row pitch C/G) that writes its 48-column
    slice of the channels-last output directly (bias, GELU, pre-activation store and the residual x in the epilogue).
    Input gradient: the same GEMM over the padded gradient with reversed taps (residual = dy). Weight gradient: one
    MN-major GEMM per group contracting over the flattened (utterance, frame) axis -- the zero padding between
    utterances removes the cross terms."""

    @staticmethod
    def forward(ctx, x, weight, bias, groups):
        x = x.contiguous()
        B, T, Cc = x.shape
        G = int(groups)
        cg = Cc // G
        k = weight.shape[2]
        assert weight.shape == (Cc, cg, k) and k % 2 == 0
        half, Tp = k // 2, T + k
        act = _resolve_act("gelu", x.dtype)
        dev, dt = x.device, x.dtype
        xg = torch.zeros((G, B, Tp, cg), dtype=dt, device=dev)
        xg[:, :, half:half + T] = x.view(B, T, G, cg).permute(2, 0, 1, 3)
        xa = _split(xg.view(G * B * Tp, cg))
        # W_f[g][co, j*cg + ci] = W[g*cg + co, ci, j]
        wf = _cast_pair(weight.detach().view(G, cg, cg, k).permute(0, 1, 3, 2).reshape(G * cg, k * cg))
        y = torch.empty_like(x)
        pre = torch.empty_like(x)
        bias_f = bias.detach().float().contiguous()
        for g in range(G):
            kw = dict(M=T, N=cg, K=k * cg, a_ld=cg, b_ld=k * cg, c_ld=Cc, nb1=B, nb2=1, a_bs=(Tp * cg, 0), b_bs=(0, 0),
                      c_bs=(T * Cc, 0))
            _passes(_off(xa, g * B * Tp * cg), _off(wf, g * cg * k * cg), y.reshape(-1)[g * cg:], kw,
                    dict(bias=bias_f[g * cg:], act=act, c_pre=pre.reshape(-1)[g * cg:],
                         residual=x.reshape(-1)[g * cg:]))
        ctx.save_for_backward(weight, pre)
        ctx.xa = xa
        ctx.meta = (B, T, Cc, G, cg, k, half, Tp, act)
        return y

    @staticmethod
    def backward(ctx, dy):
        weight, pre = ctx.saved_tensors
        B, T, Cc, G, cg, k, half, Tp, act = ctx.meta
        dev, dt = dy.device, dy.dtype
        dy = dy.contiguous()
        gq = torch.empty_like(dy)
        K.act_bwd(dy, pre, gq, act)                       # g = dy * gelu'(pre), channels-last
        dbias = torch.zeros(Cc, dtype=torch.float32, device=dev)
        K.colsum(gq.view(B * T, Cc), dbias, accumulate=True)
        front = half - 1                                  # gbuf[p] = g[p - front]
        gg = torch.zeros((G, B, Tp, cg), dtype=dt, device=dev)
        gg[:, :, front:front + T] = gq.view(B, T, G, cg).permute(2, 0, 1, 3)
        ga = _split(gg.view(G * B * Tp, cg))
        # W_b[g][ci, q*cg + co] = W[g*cg + co, ci, k-1-q]
        wb = _cast_pair(weight.detach().view(G, cg, cg, k).flip(3).permute(0, 2, 3, 1).reshape(G * cg, k * cg))
        dx = torch.empty_like(dy)
        dW2 = torch.empty((G, cg, k * cg), dtype=torch.float32, device=dev)
        Kd = B * Tp - (k - 1)                             # flattened (utterance, frame) rows with a full window
        for g in range(G):
            kw = dict(M=T, N=cg, K=k * cg, a_ld=cg, b_ld=k * cg, c_ld=Cc, nb1=B, nb2=1, a_bs=(Tp * cg, 0), b_bs=(0, 0),
                      c_bs=(T * Cc, 0))
            _passes(_off(ga, g * B * Tp * cg), _off(wb, g * cg * k * cg), dx.reshape(-1)[g * cg:], kw,
                    dict(residual=dy.reshape(-1)[g * cg:]))
            # dW2[g][co, j*cg + ci] = sum_rho gbuf_flat[rho + front, co] * xpad_flat[rho + j, ci]
            kw = dict(M=cg, N=k * cg, K=Kd, a_mn=True, b_mn=True, a_ld=cg, b_ld=cg, c_ld=k * cg)
            _passes(_off(ga, (g * B * Tp + front) * cg), _off(ctx.xa, g * B * Tp * cg), dW2[g], kw)
        dW = dW2.view(G, cg, k, cg).permute(0, 1, 3, 2).reshape(Cc, cg, k).contiguous()
        ctx.xa = None
        return dx, dW, dbias, None


# ------------------------------------------------------------------------------------------------ speech encoder prenet
def downsample_padding_mask(padding_mask, n_frames):
    """speech_encoder_prenet.py:219-229: a frame is padding iff ALL the samples it was cut from are (the samples that
    do not fill a whole frame are dropped first)."""
    extra = padding_mask.size(1) % n_frames
    if extra > 0:
        padding_mask = padding_mask[:, :-extra]
    return padding_mask.view(padding_mask.size(0), n_frames, -1).all(-1)


def padding_mask_positions(frame_padding_mask, padding_idx=1):
    """The reference feeds the BOOLEAN frame mask to the sinusoidal embedding as if it were tokens
    (speech_encoder_prenet.py:196-198 -> fairseq/utils.py:247-257 make_positions): padded frames (True == padding_idx 1)
    stay at padding_idx (the zero row), real frames count up from padding_idx + 1."""
    keep = (~frame_padding_mask).long()
    return torch.cumsum(keep, dim=1) * keep + padding_idx


class _WeightNormConv(torch.nn.Module):
    """Holds the parameters of nn.utils.weight_norm(Conv1d(d, d, k, groups), dim=2) under the reference's checkpoint
    names (`weight_g` [1, 1, k], `weight_v` [d, d/groups, k], `bias`)."""

    def __init__(self, d, k, groups):
        super().__init__()
        import math
        v = torch.empty(d, d // groups, k).normal_(0.0, math.sqrt(4.0 / (k * d)))
        self.weight_g = torch.nn.Parameter(v.norm(dim=(0, 1), keepdim=True))
        self.weight_v = torch.nn.Parameter(v)
        self.bias = torch.nn.Parameter(torch.zeros(d))
        self.groups = groups

    def weight(self):
        v = self.weight_v
        return self.weight_g * v / v.norm(dim=(0, 1), keepdim=True)


class SpeechEncoderPrenet(torch.nn.Module):
    """speech_encoder_prenet.py:57-275 for the built configuration (encoder_speech_prenet "conv", extractor_mode
    "default" or "layer_norm", use_conv_pos and use_sinc_pos as in the Base / Large archs): waveform -> [B, T, d], frame padding mask and the
    mean-square feature penalty. The HuBERT-style mask draw stays on the host (speecht5_b200.data.compute_mask_indices,
    numpy, like the reference :236-262); its result is applied here."""

    def __init__(self, args):
        super().__init__()
        from .models.modules.nets import fairseq_sinusoid_table  # noqa: F401  (table builder shared with the text prenet)
        layers = eval(args.conv_feature_layers) if isinstance(args.conv_feature_layers, str) else list(
            args.conv_feature_layers)
        if getattr(args, "encoder_speech_prenet", "conv") != "conv" or getattr(args, "use_abs_pos", False):
            raise NotImplementedError("only the conv speech prenet with conv + sinusoidal positions is built")
        if not args.use_conv_pos:  # the reference's forward needs the LayerNorm it only builds under use_conv_pos (:102-104,174)
            raise NotImplementedError("--use-conv-pos is required (as in every speech-input recipe)")
        self.embed = layers[-1][0]
        d = args.encoder_embed_dim
        # labels per frame (:89-92): label rate x total conv stride / sample rate (50 x 320 / 16000 = 1 for HuBERT labels)
        self.feat2tar_ratio = (getattr(args, "label_rates", 50) * float(np.prod([st for _, _, st in layers]))
                               / getattr(args, "sample_rate", 16000))
        self.feature_extractor = ConvFeatureExtractor(layers, args.extractor_mode, args.conv_bias)
        self.post_extract_proj = torch.nn.Linear(self.embed, d) if self.embed != d else None
        self.feature_grad_mult = args.feature_grad_mult
        self.dropout_p = args.dropout
        self.use_conv_pos, self.use_sinc_pos = args.use_conv_pos, args.use_sinc_pos
        self.padding_idx = 1
        if self.use_conv_pos:
            self.layer_norm = torch.nn.LayerNorm(self.embed)
            self.pos_conv = torch.nn.Sequential(_WeightNormConv(d, args.conv_pos, args.conv_pos_groups))
        self.mask_emb = torch.nn.Parameter(torch.empty(d).uniform_())
        self.mask_prob, self.mask_length = args.mask_prob, args.hubert_mask_length
        self.mask_selection, self.mask_other = args.mask_selection, args.mask_other
        self.no_mask_overlap, self.mask_min_space = args.no_mask_overlap, args.mask_min_space
        self._pe = None
        self.embed_dim = d
        self.freeze_encoder_updates = getattr(args, "freeze_encoder_updates", 0)
        self.num_updates = 0
        # channel masks (:253-271): prob 0.5 / length 64 in t5_transformer_base_asr (models/speecht5.py:1443-1445)
        self.mask_channel_prob = getattr(args, "mask_channel_prob", 0.0)
        self.mask_channel_length = getattr(args, "mask_channel_length", 10)
        self.mask_channel_selection = getattr(args, "mask_channel_selection", "static")
        self.mask_channel_other = getattr(args, "mask_channel_other", 0)
        self.no_mask_channel_overlap = getattr(args, "no_mask_channel_overlap", False)
        self.mask_channel_min_space = getattr(args, "mask_channel_min_space", 1)

    def _positions(self, frame_mask, B, T, device):
        if self._pe is None or self._pe.shape[0] < self.padding_idx + 1 + T or self._pe.device != device:
            from .models.modules.nets import fairseq_sinusoid_table
            self._pe = fairseq_sinusoid_table(self.padding_idx + 1 + max(T, 4000), self.embed_dim, self.padding_idx,
                                              device)
        pm = frame_mask if frame_mask is not None else torch.zeros((B, T), dtype=torch.bool, device=device)
        return self._pe.index_select(0, padding_mask_positions(pm, self.padding_idx).view(-1)).view(B, T, -1)

    def set_num_updates(self, num_updates):
        self.num_updates = num_updates

    def forward(self, src_tokens, require_feat_pen=False, target_list=None, padding_mask=None, mask=True,
                mask_indices=None, mask_channel_indices=None):
        """Reference signature and returns (speech_encoder_prenet.py:151-204): `(x, frame_padding_mask)`, or with
        require_feat_pen `((x, features_pen, mask_indices, target_list), frame_padding_mask)`. `mask_indices` [B,T] /
        `mask_channel_indices` [B,C] (extra, optional) inject a precomputed mask draw instead of sampling one here --
        the trainer draws them on the host before a CUDA-graph replay (speecht5_b200.data.draw_hubert_masks)."""
        import contextlib
        ft = self.freeze_encoder_updates <= self.num_updates
        with torch.no_grad() if not ft else contextlib.ExitStack():
            return self._forward(src_tokens, require_feat_pen, padding_mask, mask, mask_indices, mask_channel_indices,
                                 target_list)

    def forward_targets(self, features, target_list):
        """speech_encoder_prenet.py:206-217 on [B, T, C] frames: trim the frames to the span the k-means labels cover and
        pick the label of every frame (label rate x frame stride / sample rate labels per frame)."""
        feat_tsz = features.size(1)
        targ_tsz = min(t.size(1) for t in target_list)
        if self.feat2tar_ratio * feat_tsz > targ_tsz:
            feat_tsz = int(targ_tsz / self.feat2tar_ratio)
            features = features[:, :feat_tsz]
        inds = (torch.arange(feat_tsz, device=target_list[0].device).float() * self.feat2tar_ratio).long()
        return features, [t[:, inds] for t in target_list]

    def _forward(self, source, require_feat_pen, padding_mask, mask, mask_indices, mask_channel_indices=None,
                 target_list=None):
        from . import ops
        if self.feature_grad_mult > 0:
            x = self.feature_extractor(source)
            if self.feature_grad_mult != 1.0:  # GradMultiply (:156-160): identity forward, scaled gradient
                x = x * self.feature_grad_mult + x.detach() * (1.0 - self.feature_grad_mult)
        else:
            with torch.no_grad():
                x = self.feature_extractor(source)
        if target_list is not None:  # (:170-171) pre-training: frames aligned with the HuBERT labels
            x, target_list = self.forward_targets(x, target_list)
            x = x.contiguous()
        features_pen = x.float().pow(2).mean()
        B, T, _ = x.shape
        x = ops.residual_layer_norm(x, None, self.layer_norm)
        frame_mask = downsample_padding_mask(padding_mask, T) if padding_mask is not None else None
        drop = self.dropout_p if self.training else 0.0
        if self.post_extract_proj is not None:
            x = ops.linear(x, self.post_extract_proj.weight, self.post_extract_proj.bias, drop_p=drop)
        else:
            x = ops.dropout(x, drop, self.training)
        if mask and mask_indices is None and self.mask_prob > 0:  # apply_hubert_mask (:234-272): host draw, numpy
            from .data import compute_mask_indices
            mask_indices = torch.from_numpy(compute_mask_indices(
                (B, T), frame_mask.cpu() if frame_mask is not None else None, self.mask_prob, self.mask_length,
                self.mask_selection, self.mask_other, min_masks=2, no_overlap=self.no_mask_overlap,
                min_space=self.mask_min_space)).to(x.device)
        if mask and mask_channel_indices is None and self.mask_channel_prob > 0:  # second numpy draw, as :253-262
            from .data import compute_mask_indices
            mask_channel_indices = torch.from_numpy(compute_mask_indices(
                (B, x.shape[-1]), None, self.mask_channel_prob, self.mask_channel_length, self.mask_channel_selection,
                self.mask_channel_other, no_overlap=self.no_mask_channel_overlap,
                min_space=self.mask_channel_min_space)).to(x.device)
        if mask_indices is not None:
            x = torch.where(mask_indices.unsqueeze(-1), self.mask_emb.to(x.dtype), x)
        if mask_channel_indices is not None:
            x = torch.where(mask_channel_indices.unsqueeze(1), torch.zeros((), dtype=x.dtype, device=x.device), x)
        if self.use_conv_pos:
            wn = self.pos_conv[0]
            x = GroupedPosConvFn.apply(x, wn.weight(), wn.bias, wn.groups)
        if self.use_sinc_pos:
            x = x + self._positions(frame_mask, B, T, x.device).to(x.dtype)
        if require_feat_pen:
            return (x, features_pen, mask_indices, target_list), frame_mask
        return x, frame_mask


class CTCLossFn(torch.autograd.Function):
    """sum_b CTC nll of the encoder head, log-softmax fused (csrc/ctc.cu); the gradient with respect to the logits is
    produced in the same launch and scaled by the incoming scalar in backward."""

    @staticmethod
    def forward(ctx, logits, targets_flat, input_lengths, target_lengths, blank, zero_infinity):
        logits = logits.float().contiguous()
        T, B, V = logits.shape
        tl = target_lengths.long().contiguous()
        offs = (torch.cumsum(tl, 0) - tl).contiguous()
        s_max = 2 * int(tl.max().item()) + 1 if B > 0 else 1
        nll = torch.empty(B, dtype=torch.float32, device=logits.device)
        grad = torch.empty_like(logits)
        K.ctc_loss(logits, targets_flat.long().contiguous(), offs, input_lengths.long().contiguous(), tl, nll, grad,
                   s_max, int(blank), bool(zero_infinity))
        ctx.save_for_backward(grad)
        return nll.sum()

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None, None, None


def ctc_loss_sum(logits_tbv, targets_flat, input_lengths, target_lengths, blank, zero_infinity):
    return CTCLossFn.apply(logits_tbv, targets_flat, input_lengths, target_lengths, blank, zero_infinity)


class CTCLossPaddedFn(torch.autograd.Function):
    """Same kernel on right-padded targets [B, S] (row b's labels are targets[b, :target_lengths[b]]): no host sync, no
    data-dependent shapes -- the form a captured training step uses."""

    @staticmethod
    def forward(ctx, logits, targets, input_lengths, target_lengths, blank, zero_infinity):
        logits = logits.float().contiguous()
        T, B, V = logits.shape
        S = targets.size(1)
        offs = torch.arange(B, device=logits.device, dtype=torch.int64) * S
        nll = torch.empty(B, dtype=torch.float32, device=logits.device)
        grad = torch.empty_like(logits)
        K.ctc_loss(logits, targets.long().contiguous().view(-1), offs, input_lengths.long().contiguous(),
                   target_lengths.long().contiguous(), nll, grad, 2 * S + 1, int(blank), bool(zero_infinity))
        ctx.save_for_backward(grad)
        return nll.sum()

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None, None, None


def ctc_loss_sum_padded(logits_tbv, targets_bs, input_lengths, target_lengths, blank, zero_infinity):
    return CTCLossPaddedFn.apply(logits_tbv, targets_bs, input_lengths, target_lengths, blank, zero_infinity)

"""TTS criterion: mirrors speecht5/criterions/text_to_speech_loss.py (TexttoSpeechLoss :72-214, Tacotron2Loss :217-345,
GuidedMultiHeadAttentionLoss :370-427). On the device the masked reductions and their gradients are four launches of
csrc/criterion.cu (TacotronLossFn / GuidedAttnFn below) instead of ~100 elementwise ATen kernels per update; the
broadcast formulation underneath states the same arithmetic in torch ops (masks by broadcasting instead of the
reference's per-utterance Python loops, :404-413) and is what CPU tensors take and what the kernels are tested against."""
import torch
import torch.nn.functional as F

from .. import kernels as K
from ..fairseq_shim import FairseqCriterion
from ..ops import RT


def make_non_pad_mask(lengths, maxlen):
    lengths = lengths.long()
    return torch.arange(maxlen, device=lengths.device)[None, :] < lengths[:, None]


class TacotronLossFn(torch.autograd.Function):
    """(l1, l2, bce) of Tacotron2Loss with use_masking as ONE reduction pass (st5_tts_loss_fwd) and one gradient pass
    (st5_tts_loss_bwd): valid frames are l < olens - olens % r, the stop label of the last valid frame counts as 1 when
    r > 1 (text_to_speech_loss.py:161-166 + :288-330)."""

    @staticmethod
    def forward(ctx, after, before, logits, ys, labels, olens, r, pos_weight):
        after, before, logits = after.float().contiguous(), before.float().contiguous(), logits.float().contiguous()
        ys, labels, olens = ys.float(), labels.float(), olens.long().contiguous()
        if ys.stride(2) != 1 or ys.stride(1) != ys.shape[2]:
            ys = ys.contiguous()
        if labels.stride(1) != 1:
            labels = labels.contiguous()
        out = torch.empty(3, dtype=torch.float32, device=after.device)
        sums = torch.empty(K.tts_loss_ws_floats(after.shape[0], after.shape[1]), dtype=torch.float32, device=after.device)
        K.tts_loss_fwd(after, before, logits, ys, labels, olens, int(r), float(pos_weight), sums, out)
        ctx.save_for_backward(after, before, logits, ys, labels, olens, sums)
        ctx.meta = (int(r), float(pos_weight))
        return out

    @staticmethod
    def backward(ctx, g):
        after, before, logits, ys, labels, olens, sums = ctx.saved_tensors
        r, pos_weight = ctx.meta
        d_after, d_before, d_logits = torch.empty_like(after), torch.empty_like(before), torch.empty_like(logits)
        K.tts_loss_bwd(after, before, logits, ys, labels, olens, sums, g.float().contiguous(), r, pos_weight, d_after,
                       d_before, d_logits)
        return d_after, d_before, d_logits, None, None, None, None, None


class GuidedAttnFn(torch.autograd.Function):
    """GuidedMultiHeadAttentionLoss (:370-427) over the first `heads` heads of the given layers' cross-attention
    probabilities, without the torch.cat of the slices: st5_guided_attn_fwd reads the layers in place, the backward writes
    each layer's dP in the pitch the attention backward reads (heads >= `heads` are left unwritten when every producer of
    the probabilities declared that its backward never reads them, ops.attention)."""

    @staticmethod
    def forward(ctx, ilens, olens, r, heads, sigma, alpha, *atts):
        ilens, olens = ilens.long().contiguous(), olens.long().contiguous()
        heads = min(int(heads), atts[0].shape[1])  # (the reference's slice a[:, :heads] clips the same way)
        out = torch.empty(1, dtype=torch.float32, device=atts[0].device)
        gsum = torch.empty(K.guided_attn_ws_floats(len(atts), atts[0].shape[0], heads, atts[0].shape[2]),
                           dtype=torch.float32, device=atts[0].device)
        K.guided_attn_fwd(atts, int(heads), ilens, olens, int(r), float(sigma), float(alpha), gsum, out)
        ctx.save_for_backward(ilens, olens, gsum)
        sparse = all(getattr(a, "_st5_ext_heads", 0) >= heads for a in atts)
        ctx.meta = (int(r), int(heads), float(sigma), float(alpha), atts[0].shape, atts[0].stride(2), len(atts), sparse)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        ilens, olens, gsum = ctx.saved_tensors
        r, heads, sigma, alpha, (B, H, T_out, T_in), p_ld, n, sparse = ctx.meta
        datts = [torch.empty((B, H, T_out, p_ld), dtype=torch.float32, device=gsum.device) for _ in range(n)]
        K.guided_attn_bwd(datts, heads, T_in, ilens, olens, r, sigma, alpha, gsum, g.float().reshape(1).contiguous(),
                          zero_rest=not sparse)
        return (None, None, None, None, None, None) + tuple(d if p_ld == T_in else d[..., :T_in] for d in datts)


class Tacotron2Loss(torch.nn.Module):
    def __init__(self, use_masking=True, use_weighted_masking=False, bce_pos_weight=20.0):
        super().__init__()
        assert use_masking and not use_weighted_masking, "reference recipe: use_masking=True"
        self.register_buffer("pos_weight", torch.tensor(float(bce_pos_weight)), persistent=False)
        self.pos_weight_value = float(bce_pos_weight)

    def forward(self, after_outs, before_outs, logits, ys, labels, olens):
        masks = make_non_pad_mask(olens, ys.size(1)).unsqueeze(-1)
        n_el = masks.sum() * ys.size(2)
        m = masks.to(ys.dtype)
        da, db = (after_outs - ys) * m, (before_outs - ys) * m
        l1_loss = (da.abs().sum() + db.abs().sum()) / n_el
        mse_loss = ((da * da).sum() + (db * db).sum()) / n_el
        bce = F.binary_cross_entropy_with_logits(logits, labels, pos_weight=self.pos_weight.to(logits.device),
                                                 reduction="none")
        bce_loss = (bce * m[:, :, 0]).sum() / masks.sum()
        return l1_loss, mse_loss, bce_loss


class GuidedMultiHeadAttentionLoss(torch.nn.Module):
    def __init__(self, sigma=0.4, alpha=1.0):
        super().__init__()
        self.sigma, self.alpha = sigma, alpha

    def forward(self, att_ws, ilens, olens):
        """att_ws (B, H, T_out, T_in)."""
        T_out, T_in = att_ws.size(2), att_ws.size(3)
        dev = att_ws.device
        il, ol = ilens.to(dev).float(), olens.to(dev).float()
        gx = torch.arange(T_out, device=dev).float()[None, :, None] / ol[:, None, None]
        gy = torch.arange(T_in, device=dev).float()[None, None, :] / il[:, None, None]
        w = 1.0 - torch.exp(-((gy - gx) ** 2) / (2 * self.sigma ** 2))
        masks = make_non_pad_mask(olens.to(dev), T_out).unsqueeze(-1) & make_non_pad_mask(ilens.to(dev), T_in).unsqueeze(-2)
        w = (w * masks).unsqueeze(1)
        loss = (w * att_ws).sum() / (masks.sum() * att_ws.size(1))
        return self.alpha * loss


class TexttoSpeechLoss(FairseqCriterion):
    def __init__(self, task, sentence_avg=True, use_masking=True, use_weighted_masking=False, loss_type="L1",
                 bce_pos_weight=5.0, bce_loss_lambda=1.0, use_guided_attn_loss=False, guided_attn_loss_sigma=0.4,
                 guided_attn_loss_lambda=1.0, num_layers_applied_guided_attn=2, num_heads_applied_guided_attn=2,
                 modules_applied_guided_attn=("encoder-decoder",)):
        super().__init__(task)
        self.loss_type, self.bce_loss_lambda = loss_type, bce_loss_lambda
        self.use_guided_attn_loss = use_guided_attn_loss
        self.criterion = Tacotron2Loss(use_masking, use_weighted_masking, bce_pos_weight)
        self.num_heads_applied_guided_attn = num_heads_applied_guided_attn
        self.modules_applied_guided_attn = modules_applied_guided_attn
        if use_guided_attn_loss:
            self.attn_criterion = GuidedMultiHeadAttentionLoss(guided_attn_loss_sigma, guided_attn_loss_lambda)

    def forward(self, model, sample):
        net_output = model(**sample["net_input"])
        loss, l1_loss, l2_loss, bce_loss, enc_dec_attn_loss = self.compute_loss(model, net_output, sample)
        stats = torch.stack([loss.detach(), l1_loss.detach(), l2_loss.detach(), bce_loss.detach(),
                             enc_dec_attn_loss.detach() if enc_dec_attn_loss is not None else loss.new_zeros(()),
                             model.text_encoder_prenet.encoder_prenet[-1].alpha.detach().float(),
                             model.speech_decoder_prenet.decoder_prenet[-1].alpha.detach().float()])
        if getattr(self, "defer_logging", False):
            # no device->host sync inside the step (CUDA-graph capture): the caller reads `_stats` after the update
            return loss, 1, {"_stats": stats, "sample_size": 1, "ntokens": sample["ntokens"],
                             "nsentences": sample["target"].size(0)}
        stats = stats.tolist()  # the reference's ~7 .item() calls (:129-146) batched into ONE device->host copy
        logging_output = {"loss": stats[0], "l1_loss": stats[1], "l2_loss": stats[2], "bce_loss": stats[3],
                          "sample_size": 1, "ntokens": sample["ntokens"], "nsentences": sample["target"].size(0)}
        if enc_dec_attn_loss is not None:
            logging_output["enc_dec_attn_loss"] = stats[4]
        logging_output["encoder_alpha"], logging_output["decoder_alpha"] = stats[5], stats[6]
        return loss, 1, logging_output

    def compute_loss(self, model, net_output, sample):
        before_outs, after_outs, logits, attn = net_output
        labels, ys = sample["labels"], sample["dec_target"]
        olens, ilens = sample["dec_target_lengths"], sample["src_lengths"]
        r = model.reduction_factor
        fused = after_outs.is_cuda  # device tensors always take the C-ABI kernels (no torch fallback on the GPU)
        if fused:
            # masks, the forced stop label of the last frame and olens - olens % r are applied inside the kernel
            l1_loss, l2_loss, bce_loss = TacotronLossFn.apply(after_outs, before_outs, logits, ys, labels, olens, r,
                                                              self.criterion.pos_weight_value).unbind(0)
            olens_in = None
        else:
            if r > 1:
                olens_in = torch.div(olens, r, rounding_mode="floor")
                olens = olens - olens % r
                # The reference slices ys/labels to max(olens) (:161-166); frames beyond it are masked out anyway, so we
                # keep the padded length (= the model output length) and avoid a device->host sync in the step.
                L = after_outs.size(1)
                ys, labels = ys[:, :L], labels[:, :L]
                labels = torch.scatter(labels, 1, (olens - 1).unsqueeze(1), 1.0)
            else:
                olens_in = olens
            l1_loss, l2_loss, bce_loss = self.criterion(after_outs, before_outs, logits, ys, labels, olens)
        if self.loss_type == "L1":
            loss = l1_loss + self.bce_loss_lambda * bce_loss if self.bce_loss_lambda > 0.0 else l1_loss
        elif self.loss_type == "L2":
            loss = l2_loss + self.bce_loss_lambda * bce_loss if self.bce_loss_lambda > 0.0 else l2_loss
        elif self.loss_type == "L1+L2":
            loss = l1_loss + l2_loss + self.bce_loss_lambda * bce_loss if self.bce_loss_lambda > 0.0 else l1_loss + l2_loss
        else:
            raise ValueError("unknown --loss-type " + self.loss_type)
        enc_dec_attn_loss = None
        if self.use_guided_attn_loss and "encoder-decoder" in self.modules_applied_guided_attn:
            if sample.get("task_name") == "s2s" and getattr(model, "speech_encoder_prenet", None) is not None:
                # (:198-206) a waveform source: the encoder sees the conv front end's frames, not the samples
                ilens = model.speech_encoder_prenet.get_src_lengths(ilens)
            attn = list(attn) if isinstance(attn, (list, tuple)) else [attn]
            if fused:
                enc_dec_attn_loss = GuidedAttnFn.apply(ilens, sample["dec_target_lengths"], r,
                                                       self.num_heads_applied_guided_attn, self.attn_criterion.sigma,
                                                       self.attn_criterion.alpha, *attn)
            else:
                att_ws = torch.cat([a[:, : self.num_heads_applied_guided_attn] for a in attn], dim=1)
                enc_dec_attn_loss = self.attn_criterion(att_ws, ilens, olens_in)
            loss = loss + enc_dec_attn_loss
        return loss, l1_loss, l2_loss, bce_loss, enc_dec_attn_loss

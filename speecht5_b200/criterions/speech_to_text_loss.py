"""Speech-to-text criterion: behaviour of speecht5/criterions/speech_to_text_loss.py (SpeechtoTextLoss :113-337,
label_smoothed_nll_loss :93-110) for the opt-in speech-input branch. The arithmetic acts on vocabulary-sized tensors
([B, T_d, V] decoder logits, [T_e, B, V] CTC head) and is issued as torch library calls (log_softmax, gather,
on CPU tensors F.ctc_loss with cuDNN off like the reference :326; on the device csrc/ctc.cu through
frontend.ctc_loss_sum / ctc_loss_sum_padded, whose recursion is specified in tests/test_kernel_algorithms_cpu.py)."""

import torch
import torch.nn.functional as F

from ..fairseq_shim import FairseqCriterion


def label_smoothed_nll_loss(lprobs, target, epsilon, ignore_index=None, reduce=True):
    """:93-110. lprobs [N, V], target [N]; note the reference's weights: (1 - eps - eps/(V-1)) nll + eps/(V-1) smooth."""
    target = target.unsqueeze(-1)
    nll = -lprobs.gather(dim=-1, index=target)
    smooth = -lprobs.sum(dim=-1, keepdim=True)
    if ignore_index is not None:
        keep = target.ne(ignore_index)
        nll, smooth = nll * keep, smooth * keep
    if reduce:
        nll, smooth = nll.sum(), smooth.sum()
    eps_i = epsilon / (lprobs.size(-1) - 1)
    return (1.0 - epsilon - eps_i) * nll + eps_i * smooth, nll


def _edit_distance(a, b):
    """Levenshtein distance between two sequences (the reference imports `editdistance` for its eval-time error counts)."""
    prev = list(range(len(b) + 1))
    for i, x in enumerate(a, 1):
        cur = [i]
        for j, y in enumerate(b, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (x != y)))
        prev = cur
    return prev[-1]


class SpeechtoTextLoss(FairseqCriterion):
    def __init__(self, task, sentence_avg=True, label_smoothing=0.1, ignore_prefix_size=0, report_accuracy=False,
                 ce_weight=1.0, ctc_weight=0.0, zero_infinity=False, post_process="sentencepiece"):
        super().__init__(task)
        d = getattr(task, "target_dictionary", None)
        self.blank_idx = d.index(task.blank_symbol) if (d is not None and hasattr(task, "blank_symbol")) else 0  # :127-131
        self.pad_idx = d.pad() if d is not None else 1
        self.eos_idx = d.eos() if d is not None else 2
        self.padding_idx = self.pad_idx
        self.sentence_avg, self.eps = sentence_avg, label_smoothing
        self.ignore_prefix_size, self.report_accuracy = ignore_prefix_size, report_accuracy
        self.ce_weight, self.ctc_weight = ce_weight, ctc_weight
        self.zero_infinity, self.post_process = zero_infinity, post_process
        if ce_weight <= 0 and ctc_weight <= 0:
            raise ValueError("SpeechtoTextLoss: ce_weight or ctc_weight must be positive")

    # ------------------------------------------------------------------ cross entropy on the decoder (:340-372)
    def get_lprobs_and_target(self, model, net_output, sample):
        lprobs = model.get_normalized_probs(net_output, log_probs=True)
        target = model.get_targets(sample, net_output)
        if self.ignore_prefix_size > 0:
            if getattr(lprobs, "batch_first", False):
                lprobs, target = lprobs[:, self.ignore_prefix_size:], target[:, self.ignore_prefix_size:]
            else:
                lprobs, target = lprobs[self.ignore_prefix_size:], target[self.ignore_prefix_size:]
        return lprobs.reshape(-1, lprobs.size(-1)), target.reshape(-1)

    def compute_loss(self, model, net_output, sample, reduce=True):
        lprobs, target = self.get_lprobs_and_target(model, net_output, sample)
        return label_smoothed_nll_loss(lprobs, target, self.eps, ignore_index=self.padding_idx, reduce=reduce)

    def compute_accuracy(self, model, net_output, sample):
        lprobs, target = self.get_lprobs_and_target(model, net_output, sample)
        mask = target.ne(self.padding_idx)
        return (lprobs.argmax(1).eq(target) & mask).sum(), mask.sum()

    # ------------------------------------------------------------------ CTC on the encoder head (:303-335)
    def compute_loss_ctc(self, model, net_output, sample):
        lprobs = model.get_normalized_probs_for_ctc(net_output, log_probs=True).contiguous()  # [T, B, V]
        pm = net_output["encoder_padding_mask"]
        if pm is not None and len(pm) > 0 and pm[0] is not None:
            input_lengths = (~pm[0]).long().sum(-1)
        else:
            input_lengths = lprobs.new_full((lprobs.size(1),), lprobs.size(0), dtype=torch.long)
        keep = (sample["target"] != self.pad_idx) & (sample["target"] != self.eos_idx)
        target_lengths = (sample["target_lengths"] if "target_lengths" in sample else keep.sum(-1)) - 1  # :324
        targets_flat = None if getattr(self, "defer_logging", False) else sample["target"].masked_select(keep)
        raw = net_output["encoder_out_for_ctc"][0]
        if getattr(self, "defer_logging", False) and raw.is_cuda:
            # captured step (B200Trainer): padded targets straight into the fused log-softmax + CTC kernel, lengths
            # read on the device. Collated targets are right-padded tokens + eos + pad (:316-324 keeps the first
            # target_lengths - 1 of each row, which is what masked_select(keep) concatenates)
            from ..frontend import ctc_loss_sum_padded
            loss = ctc_loss_sum_padded(raw, sample["target"], input_lengths, target_lengths, self.blank_idx,
                                       self.zero_infinity)
            return loss, lprobs, input_lengths
        if raw.is_cuda:  # device tensors always take csrc/ctc.cu (fused log-softmax + CTC + logit gradient)
            from ..frontend import ctc_loss_sum
            loss = ctc_loss_sum(raw, targets_flat, input_lengths, target_lengths, self.blank_idx, self.zero_infinity)
            return loss, lprobs, input_lengths
        with torch.backends.cudnn.flags(enabled=False):
            loss = F.ctc_loss(lprobs, targets_flat, input_lengths, target_lengths, blank=self.blank_idx,
                              reduction="sum", zero_infinity=self.zero_infinity)
        return loss, lprobs, input_lengths

    # ------------------------------------------------------------------ speaker identification (s2c)
    def _forward_s2c(self, model, sample):
        """speecht5_criterion.py:113 sends s2c here: the model returns ((class logits [B, N], embedding), None) and the
        loss is the label-smoothed CE of compute_loss on target [B, 1], with compute_accuracy's counts; one row kernel
        (csrc/speaker_head.cu) computes all of it. The speaker model has no CTC head."""
        from .. import ops
        if self.ctc_weight > 0 or self.ce_weight <= 0:
            raise NotImplementedError("speaker identification is trained with cross entropy only (ctc_weight 0)")
        (logits, _), _ = model(**sample["net_input"])
        sums = ops.margin_ce(logits, sample["target"], self.eps, self.padding_idx)  # loss, nll, n_correct, total
        loss, nll = sums[0], sums[1]
        ntokens = sample["ntokens"] if "ntokens" in sample else int(sample["target_lengths"].sum().item())
        sample_size = sample["target"].size(0) if self.sentence_avg else ntokens
        nsent = sample["target"].size(0)
        if getattr(self, "defer_logging", False):
            stats = torch.stack([loss.detach(), loss.detach(), loss.new_zeros(()), nll.detach(), sums[2], sums[3]])
            return loss, sample_size, {"_stats": stats, "ntokens": ntokens, "nsentences": nsent,
                                       "sample_size": sample_size}
        log = {"loss": loss.item(), "ce_loss": loss.item(), "ctc_loss": 0, "nll_loss": nll.item(), "ntokens": ntokens,
               "nsentences": nsent, "sample_size": sample_size}
        if self.report_accuracy:
            log["n_correct"], log["total"] = int(sums[2].item()), int(sums[3].item())
        return loss, sample_size, log

    def forward(self, model, sample, reduce=True):
        if sample.get("task_name") == "s2c" and getattr(model, "speaker_decoder_postnet", None) is not None:
            return self._forward_s2c(model, sample)
        if self.ce_weight == 0 and self.ctc_weight > 0:
            sample["only_ctc"] = True  # (:189-190; as in the reference this key never reaches the model call)
        net_output_decoder, net_output = model(**sample["net_input"])
        loss_ce = nll = loss_ctc = None
        if self.ce_weight > 0:
            loss_ce, nll = self.compute_loss(model, net_output_decoder, sample, reduce=reduce)
        if self.ctc_weight > 0:
            loss_ctc, lprobs, input_lengths = self.compute_loss_ctc(model, net_output, sample)
        if loss_ce is not None and loss_ctc is not None:
            loss = self.ce_weight * loss_ce + self.ctc_weight * loss_ctc
        else:
            loss = loss_ce if loss_ce is not None else loss_ctc  # a single term is NOT scaled by its weight (:202-205)
        ntokens = sample["ntokens"] if "ntokens" in sample else int(sample["target_lengths"].sum().item())
        sample_size = sample["target"].size(0) if self.sentence_avg else ntokens
        if getattr(self, "defer_logging", False):
            # no device->host sync inside the step (CUDA-graph capture): the caller reads `_stats` after the update
            z = loss.new_zeros(())
            stats = torch.stack([loss.detach(), loss_ce.detach() if loss_ce is not None else z,
                                 loss_ctc.detach() if loss_ctc is not None else z, nll.detach() if nll is not None else z])
            return loss, sample_size, {"_stats": stats, "ntokens": ntokens, "nsentences": sample["target"].size(0),
                                       "sample_size": sample_size}
        log = {"loss": loss.item(), "ce_loss": loss_ce.item() if loss_ce is not None else 0,
               "ctc_loss": loss_ctc.item() if loss_ctc is not None else 0, "nll_loss": nll.item() if nll is not None else 0,
               "ntokens": ntokens, "nsentences": sample["target"].size(0), "sample_size": sample_size}
        if loss_ce is not None and self.report_accuracy:
            n_correct, total = self.compute_accuracy(model, net_output_decoder, sample)
            log["n_correct"], log["total"] = int(n_correct.item()), int(total.item())
        if loss_ctc is not None and not model.training:  # greedy CTC unit error counts (:232-300; no external LM)
            with torch.no_grad():
                best = lprobs.argmax(-1).transpose(0, 1).cpu()  # [B, T]
                tgt = (sample["target_label"] if "target_label" in sample else sample["target"]).cpu()
                c_err = c_len = 0
                for hyp, t, n in zip(best, tgt, input_lengths.tolist()):
                    ref = t[(t != self.pad_idx) & (t != self.eos_idx)].tolist()
                    toks = torch.unique_consecutive(hyp[:n])
                    c_err += _edit_distance(toks[toks != self.blank_idx].tolist(), ref)
                    c_len += len(ref)
                log["c_errors"], log["c_total"] = c_err, c_len
        return loss, sample_size, log

    @staticmethod
    def logging_outputs_can_be_summed() -> bool:
        return True

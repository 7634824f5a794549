"""@register_criterion("speecht5") dispatcher, mirroring speecht5/criterions/speecht5_criterion.py:23-120: routes on
sample['task_name'] to the t2s / s2s (TexttoSpeechLoss), s2t and s2c (SpeechtoTextLoss), text_pretrain and speech_pretrain
criteria; note the reference dispatcher does not forward guided_attn_loss_lambda, so the effective guided-attention
weight is 1.0 (speecht5_criterion.py:61-71)."""
import math
import re
from dataclasses import dataclass, field

from ..fairseq_shim import FairseqCriterion, metrics, register_criterion
from .speech_pretrain_criterion import SpeechPretrainCriterion
from .speech_to_text_loss import SpeechtoTextLoss
from .text_pretrain_criterion import TextPretrainCriterion
from .text_to_speech_loss import TexttoSpeechLoss


@dataclass
class SpeechT5CriterionConfig:
    """Union of the reference's criterion configs (speecht5_criterion.py:23-30 inherits the text-to-speech,
    speech-to-text, label-smoothed CE and pre-training configs), so every recipe's `--criterion speecht5 ...` flags
    parse."""
    sentence_avg: bool = field(default=True)
    # text_to_speech_loss.py:21-69
    use_masking: bool = field(default=True)
    use_weighted_masking: bool = field(default=False)
    loss_type: str = field(default="L1")
    bce_pos_weight: float = field(default=5.0)
    bce_loss_lambda: float = field(default=1.0)
    use_guided_attn_loss: bool = field(default=False)
    guided_attn_loss_sigma: float = field(default=0.4)
    guided_attn_loss_lambda: float = field(default=10.0)
    num_layers_applied_guided_attn: int = field(default=2)
    num_heads_applied_guided_attn: int = field(default=2)
    # speech_to_text_loss.py:27-91 / label-smoothed CE
    zero_infinity: bool = field(default=False)
    post_process: str = field(default="sentencepiece")
    label_smoothing: float = field(default=0.0)
    report_accuracy: bool = field(default=False)
    ignore_prefix_size: int = field(default=0)
    ce_weight: float = field(default=1.0)
    ctc_weight: float = field(default=0.0)
    # pre-training criteria (speech_pretrain_criterion.py, text_pretrain_criterion.py)
    pred_masked_weight: float = field(default=1.0)
    pred_nomask_weight: float = field(default=0.0)
    # (the reference dataclass inherits the text criterion's default for the shared list, the recipes pass [10, 0.1])
    loss_weights: list = field(default_factory=lambda: [0.1])
    log_keys: list = field(default_factory=list)
    dec_weight: float = field(default=1.0)
    bart_weight: float = field(default=1.0)
    hubert_weight: float = field(default=1.0)


@register_criterion("speecht5", dataclass=SpeechT5CriterionConfig)
class SpeechT5Criterion(FairseqCriterion):
    def __init__(self, task, sentence_avg=True, use_masking=True, loss_type="L1", bce_pos_weight=5.0,
                 bce_loss_lambda=1.0, use_guided_attn_loss=False, guided_attn_loss_sigma=0.4,
                 num_heads_applied_guided_attn=2, label_smoothing=0.0, ignore_prefix_size=0, report_accuracy=False,
                 ce_weight=1.0, ctc_weight=0.0, zero_infinity=False, post_process="sentencepiece", pred_masked_weight=1.0,
                 pred_nomask_weight=0.0, loss_weights=(10.0,), log_keys=None, use_weighted_masking=False,
                 hubert_weight=1.0, dec_weight=1.0, bart_weight=1.0, **unused):
        super().__init__(task)
        self.text_to_speech_loss = TexttoSpeechLoss(
            task, sentence_avg, use_masking, False, loss_type, bce_pos_weight, bce_loss_lambda, use_guided_attn_loss,
            guided_attn_loss_sigma, 1.0, 2, num_heads_applied_guided_attn)
        # s2t branch (speecht5_criterion.py:72-81); meaningful only with the opt-in speech-input / text-output model
        self.speech_to_text_loss = SpeechtoTextLoss(task, sentence_avg, label_smoothing, ignore_prefix_size,
                                                    report_accuracy, ce_weight, ctc_weight, zero_infinity, post_process)
        # pre-training branches (speecht5_criterion.py:82-101): both share the configured loss_weights list
        self.text_pretrain_criterion = TextPretrainCriterion(task, sentence_avg, bart_weight, loss_weights)
        self.speech_pretrain_criterion = SpeechPretrainCriterion(
            task, sentence_avg, pred_masked_weight, pred_nomask_weight, loss_weights, log_keys, use_masking,
            use_weighted_masking, loss_type, bce_pos_weight, hubert_weight, dec_weight)

    def forward(self, model, sample, reduce=True):
        task_name = sample["task_name"]
        if task_name in ("t2s", "s2s"):
            return self.text_to_speech_loss(model, sample)
        if task_name in ("s2t", "s2c"):  # (:113: speaker identification is CE on the class logits)
            return self.speech_to_text_loss(model, sample, reduce)
        if task_name == "text_pretrain":
            return self.text_pretrain_criterion(model, sample, reduce)
        if task_name == "speech_pretrain":
            return self.speech_pretrain_criterion(model, sample, reduce)
        raise NotImplementedError(f"criterion branch '{task_name}' is not built in the H100 path")

    # ------------------------------------------------------------------ logging (speecht5_criterion.py:123-436)
    @staticmethod
    def _sum(logs, key):
        return sum(log.get(key, 0) for log in logs)

    @classmethod
    def reduce_metrics(cls, logging_outputs):
        """Aggregate the per-rank / per-micro-batch logging outputs (each {task_name: criterion log, "loss": ...,
        "sample_size": 1}, the shape `SpeechT5Task.train_step` returns, tasks/speecht5.py:519-556) into fairseq's meters
        under the reference's key names: t2s_* / s2s_* (:226-255, :281-308), s2t_* with ctc_loss / ce_loss / accuracy /
        uer / wer (:137-224), text_* / bart_* (:310-346), hubert_* (:348-417) and the overall "loss" (:419-423)."""
        by_task = {}
        for log in logging_outputs:
            for task_name, val in log.items():
                if task_name in ("s2t", "t2s", "s2c", "s2s", "text_pretrain", "speech_pretrain"):
                    by_task.setdefault(task_name, []).append(val)
        S, ln2 = cls._sum, math.log(2)
        for task_name, logs in by_task.items():
            sample_size = max(1, S(logs, "sample_size"))
            ntokens = S(logs, "ntokens")
            if task_name in ("s2t", "s2c"):
                metrics.log_scalar(f"{task_name}_loss", S(logs, "loss") / sample_size / ln2, sample_size, 1, round=3)
                metrics.log_scalar(f"{task_name}_nll_loss", S(logs, "nll_loss") / ntokens / ln2, ntokens, 2, round=3)
                if task_name == "s2t":
                    metrics.log_derived("s2t_ppl", lambda meters: _perplexity(meters["s2t_nll_loss"].avg, 2))
                    metrics.log_scalar("ctc_loss", S(logs, "ctc_loss") / sample_size / ln2, ntokens, 2, round=3)
                    metrics.log_scalar("ce_loss", S(logs, "ce_loss") / ntokens, ntokens, 2, round=3)
                total = _item(S(logs, "total"))
                if total > 0:
                    metrics.log_scalar(f"{task_name}_total", total)
                    metrics.log_scalar(f"{task_name}_n_correct", _item(S(logs, "n_correct")))
                    metrics.log_derived(
                        f"{task_name}_accuracy",
                        lambda meters, t=task_name: round(meters[f"{t}_n_correct"].sum * 100.0 / meters[f"{t}_total"].sum, 3)
                        if meters[f"{t}_total"].sum > 0 else float("nan"), 2)
                if task_name == "s2t":
                    for k in ("c_errors", "c_total", "w_errors", "wv_errors", "w_total"):
                        metrics.log_scalar("_" + k, S(logs, k))
                    if S(logs, "c_total") > 0:
                        metrics.log_derived("uer", lambda meters: _ratio(meters, "_c_errors", "_c_total"))
                    if S(logs, "w_total") > 0:
                        metrics.log_derived("wer", lambda meters: _ratio(meters, "_w_errors", "_w_total"))
                        metrics.log_derived("raw_wer", lambda meters: _ratio(meters, "_wv_errors", "_w_total"))
            elif task_name in ("t2s", "s2s"):
                t = task_name
                metrics.log_scalar(f"{t}_loss", S(logs, "loss") / sample_size, sample_size, 1, round=5)
                for k in ("l1_loss", "l2_loss", "bce_loss"):
                    metrics.log_scalar(f"{t}_{k}", S(logs, k) / sample_size, sample_size, 2, round=5)
                if t == "t2s":
                    metrics.log_scalar("t2s_encoder_alpha", S(logs, "encoder_alpha") / sample_size, sample_size, round=5)
                metrics.log_scalar(f"{t}_decoder_alpha", S(logs, "decoder_alpha") / sample_size, sample_size, round=5)
                if "enc_dec_attn_loss" in logs[0]:
                    metrics.log_scalar(f"{t}_enc_dec_attn_loss", S(logs, "enc_dec_attn_loss") / sample_size, sample_size,
                                       round=8)
            elif task_name == "text_pretrain":
                bart = S(logs, "bart_loss")
                metrics.log_scalar("text_loss", S(logs, "loss") / sample_size / ln2, sample_size, round=3)
                metrics.log_scalar("bart_loss", bart / sample_size / ln2, ntokens, 2, round=3)
                if sample_size != ntokens:
                    metrics.log_scalar("bart_nll_loss", bart / ntokens / ln2, ntokens, round=3)
                    metrics.log_derived("bart_ppl", lambda meters: _perplexity(meters["bart_nll_loss"].avg))
                else:
                    metrics.log_derived("bart_ppl", lambda meters: _perplexity(meters["bart_loss"].avg))
                metrics.log_scalar("bart_wpb", ntokens, priority=180, round=1)
                cls._log_perplexities(logs, "text")
            elif task_name == "speech_pretrain":
                ngpu = S(logs, "ngpu")
                loss_sum = S(logs, "loss")
                metrics.log_scalar("hubert_loss", loss_sum / sample_size / ln2, sample_size, round=3)
                if sample_size != ntokens:
                    metrics.log_scalar("hubert_nll_loss", loss_sum / ntokens / ln2, ntokens, round=3)
                    metrics.log_derived("hubert_ppl", lambda meters: _perplexity(meters["hubert_nll_loss"].avg))
                else:
                    metrics.log_derived("hubert_ppl", lambda meters: _perplexity(meters["hubert_loss"].avg))
                counts = {}
                for lk in logs[0]:
                    if lk.startswith("count_"):
                        counts[lk] = S(logs, lk)
                        metrics.log_scalar("hubert_" + lk, counts[lk])
                for lk in logs[0]:
                    if lk.startswith("loss_") and lk != "loss_prob_perplexity":
                        metrics.log_scalar("hubert_" + lk, S(logs, lk) / sample_size / ln2, round=3)
                    elif lk.startswith("correct_"):
                        metrics.log_scalar("hubert_" + lk, S(logs, lk) / counts[re.sub("correct", "count", lk)])
                cls._log_perplexities(logs, "hubert")
                for k in ("dec_loss", "l1_loss", "l2_loss", "bce_loss"):
                    metrics.log_scalar("hubert_" + k, S(logs, k) / ngpu, sample_size, 2, round=5)
                if "enc_dec_attn_loss" in logs[0]:
                    metrics.log_scalar("hubert_enc_dec_attn_loss", S(logs, "enc_dec_attn_loss") / ngpu, sample_size, round=8)
                metrics.log_scalar("hubert_wpb", ntokens, priority=180, round=1)
        total_size = max(1, S(logging_outputs, "sample_size"))
        metrics.log_scalar("loss", S(logging_outputs, "loss") / total_size, total_size, 1, round=5)

    @staticmethod
    def _log_perplexities(logs, prefix):
        pp = sum(log["loss_prob_perplexity"] for log in logs if "loss_prob_perplexity" in log)
        pp_size = sum(log["sample_size"] for log in logs if "loss_prob_perplexity" in log)
        cp = [log["code_perplexity"] for log in logs if "code_perplexity" in log]
        if pp > 0:
            metrics.log_scalar(f"{prefix}_loss_prob_perplexity", pp / pp_size / math.log(2), round=3)
        if sum(cp) > 0:
            metrics.log_scalar(f"{prefix}_code_perplexity", sum(cp) / len(cp), round=3)

    @staticmethod
    def logging_outputs_can_be_summed() -> bool:
        return False


def _item(x):
    return x.item() if hasattr(x, "item") else x


def _perplexity(loss, round_=2, base=2):  # fairseq/utils.py:506-515 get_perplexity
    if loss is None:
        return 0.0
    try:
        return round(base ** loss, round_)
    except OverflowError:
        return float("inf")


def _ratio(meters, num, den):
    return round(meters[num].sum * 100.0 / meters[den].sum, 3) if meters[den].sum > 0 else float("nan")

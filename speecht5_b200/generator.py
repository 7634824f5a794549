"""The generator object fairseq's `generate.py` drives (`task.build_generator(models, args)` ->
`task.inference_step(generator, models, sample)` -> `generator.generate(models, sample)`), for beam size 1: the search of
speecht5/sequence_generator.py:207-655 with ctc_weight 0 and no LM is `T5TransformerModel.generate_text_greedy`; this
class gives it the SequenceGenerator call / return shape (:191-205, :596-655: a list over sentences of a list over beams
of {"tokens", "score", "attention", "alignment", "positional_scores"}, score = sum of the token log-probabilities
divided by length ** len_penalty when normalize_scores is on). Beam search > 1, LM fusion and CTC rescoring are out of
scope (SURVEY section 2) and raise."""
import torch


class GreedyGenerator:
    def __init__(self, models, tgt_dict, beam_size=1, max_len_a=0, max_len_b=200, min_len=1, normalize_scores=True,
                 len_penalty=1.0, unk_penalty=0.0, temperature=1.0, ctc_weight=0.0, lm_model=None, use_cache=True,
                 blank=None, mask_idx=None, **unused):
        if beam_size != 1:
            raise NotImplementedError("beam search > 1 is not built in the H100 path (SURVEY section 2): use --beam 1")
        if ctc_weight and ctc_weight > 0 or lm_model is not None:
            raise NotImplementedError("CTC rescoring / LM fusion are not built in the H100 path")
        self.model = models[0] if isinstance(models, (list, tuple)) else models
        self.tgt_dict = tgt_dict
        self.pad, self.eos, self.unk = tgt_dict.pad(), tgt_dict.eos(), tgt_dict.unk()
        self.max_len_a, self.max_len_b, self.min_len = max_len_a, max_len_b, min_len
        self.normalize_scores, self.len_penalty = normalize_scores, len_penalty
        self.unk_penalty, self.temperature, self.use_cache = unk_penalty, temperature, use_cache
        index = getattr(tgt_dict, "index", None)
        self.blank = blank if blank is not None else (index("<ctc_blank>") if index else 0)
        self.mask_idx = mask_idx if mask_idx is not None else (index("<mask>") if index else None)

    @torch.no_grad()
    def generate(self, models, sample, prefix_tokens=None, constraints=None, bos_token=None):
        if prefix_tokens is not None or constraints is not None:
            raise NotImplementedError("prefix tokens / constraints are not built for the greedy path")
        ni = sample["net_input"]
        hyp, scores = self.model.generate_text_greedy(
            ni["source"], ni.get("padding_mask"), max_len_a=self.max_len_a, max_len_b=self.max_len_b, min_len=self.min_len,
            unk_penalty=self.unk_penalty, temperature=self.temperature, pad=self.pad, eos=self.eos, unk=self.unk,
            blank=self.blank, mask_idx=self.mask_idx, use_cache=self.use_cache, return_scores=True)
        out = []
        for tok, pos in zip(hyp, scores):
            total = pos.sum()
            if self.normalize_scores:
                total = total / (len(tok) ** self.len_penalty)
            out.append([{"tokens": tok, "score": total, "attention": None, "alignment": torch.empty(0),
                         "positional_scores": pos}])
        return out

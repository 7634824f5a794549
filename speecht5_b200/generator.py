"""The generator object fairseq's `generate.py` drives (`task.build_generator(models, args)` ->
`task.inference_step(generator, models, sample)` -> `generator.generate(models, sample)`), for beam size 1: the search of
speecht5/sequence_generator.py:207-655 with ctc_weight 0 and no LM is `T5TransformerModel.generate_text_greedy`; this
class gives it the SequenceGenerator call / return shape (:191-205, :596-655: a list over sentences of a list over beams
of {"tokens", "score", "attention", "alignment", "positional_scores"}, score = sum of the token log-probabilities
divided by length ** len_penalty when normalize_scores is on). Beam search > 1 is BeamSearchGenerator
(`task.build_generator(models, args, seq_gen_cls=BeamSearchGenerator)`). LM fusion (`lm_model` / `lm_weight`, what
generate.py passes for --lm-path / --lm-weight) runs on the beam path at every beam size, beam 1 included; CTC rescoring
is out of scope (SURVEY section 2) and raises."""
import torch


def _fusion_lm(lm_model):
    if lm_model is None:
        return None
    from .lm import TransformerLM
    return TransformerLM.from_fairseq(lm_model)


class GreedyGenerator:
    def __init__(self, models, tgt_dict, beam_size=1, max_len_a=0, max_len_b=200, min_len=1, normalize_scores=True,
                 len_penalty=1.0, unk_penalty=0.0, temperature=1.0, ctc_weight=0.0, lm_model=None, lm_weight=1.0,
                 use_cache=True, blank=None, mask_idx=None, **unused):
        if beam_size != 1:
            raise NotImplementedError("beam search > 1 is not built in the H100 path (SURVEY section 2): use --beam 1")
        if ctc_weight and ctc_weight > 0:
            raise NotImplementedError("CTC rescoring is not built in the H100 path")
        # with an LM the reference runs its beam search at beam 1 too: BeamSearchGenerator, K = 1
        self.lm, self.lm_weight = _fusion_lm(lm_model), lm_weight
        self.beam = None if self.lm is None else BeamSearchGenerator(models, tgt_dict, beam_size=1, max_len_a=max_len_a,
                                                                      max_len_b=max_len_b, min_len=min_len,
                                                                      normalize_scores=normalize_scores,
                                                                      len_penalty=len_penalty, unk_penalty=unk_penalty,
                                                                      temperature=temperature, lm_model=self.lm,
                                                                      lm_weight=lm_weight, use_cache=use_cache,
                                                                      blank=blank, mask_idx=mask_idx)
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
        if self.beam is not None:
            return self.beam.generate(models, sample, prefix_tokens=prefix_tokens, constraints=constraints,
                                      bos_token=bos_token)
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


class BeamSearchGenerator:
    """The SequenceGenerator of sequence_generator.py:207-654 for beam_size K >= 2, or any K with a language model
    (ctc_weight 0, no prefix tokens or constraints) on T5TransformerModel.generate_text_beam; same keywords as
    GreedyGenerator. lm_model / lm_weight: shallow fusion (:420-426) with a speecht5_b200.lm.TransformerLM or the fairseq
    transformer_lm generate.py loads from --lm-path. beam_size 1 without an LM is GreedyGenerator itself. use_cache: True
    (eager step body) or "graph" (one captured CUDA graph per step)."""

    def __init__(self, models, tgt_dict, beam_size=5, max_len_a=0, max_len_b=200, min_len=1, normalize_scores=True,
                 len_penalty=1.0, unk_penalty=0.0, temperature=1.0, ctc_weight=0.0, lm_model=None, lm_weight=1.0,
                 use_cache=True, blank=None, mask_idx=None, **unused):
        kw = dict(max_len_a=max_len_a, max_len_b=max_len_b, min_len=min_len, normalize_scores=normalize_scores,
                  len_penalty=len_penalty, unk_penalty=unk_penalty, temperature=temperature, ctc_weight=ctc_weight,
                  use_cache=use_cache, blank=blank, mask_idx=mask_idx)
        # (GreedyGenerator checks the options this class shares with it: CTC weight)
        self.greedy = GreedyGenerator(models, tgt_dict, beam_size=1, **kw)
        self.lm, self.lm_weight = _fusion_lm(lm_model), float(lm_weight)
        self.beam_size = int(beam_size)
        if (self.beam_size != 1 or self.lm is not None) and use_cache not in (True, "graph"):
            raise ValueError(f"beam search runs with use_cache=True or 'graph', got {use_cache!r}")

    @torch.no_grad()
    def generate(self, models, sample, prefix_tokens=None, constraints=None, bos_token=None):
        g = self.greedy
        if self.beam_size == 1 and self.lm is None:
            return g.generate(models, sample, prefix_tokens=prefix_tokens, constraints=constraints, bos_token=bos_token)
        if prefix_tokens is not None or constraints is not None:
            raise NotImplementedError("prefix tokens / constraints are not built for beam search")
        ni = sample["net_input"]
        return g.model.generate_text_beam(
            ni["source"], ni.get("padding_mask"), beam_size=self.beam_size, max_len_a=g.max_len_a,
            max_len_b=g.max_len_b, min_len=g.min_len, unk_penalty=g.unk_penalty, temperature=g.temperature, pad=g.pad,
            eos=g.eos, unk=g.unk, blank=g.blank, mask_idx=g.mask_idx, use_cache=g.use_cache,
            normalize_scores=g.normalize_scores, len_penalty=g.len_penalty, lm=self.lm, lm_weight=self.lm_weight)

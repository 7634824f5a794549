"""Statement of st5_beam_topk_lm (LM shallow fusion, speecht5/sequence_generator.py:420-455), written from those
semantics next to tests/beam_ref.py, which states st5_beam_topk:

* `fused_lprobs` -- per row, log_softmax(x / T) + lm_weight * log_softmax(y) on the first V_lm entries (no temperature on
                    the LM), then the masking of beam_ref.masked_lprobs in the reference's order (eos ban, NaN -> -inf,
                    mask, max_len); any dtype (float64 for kernel checks, float32 for parity).
* `topk`         -- each sentence's best min(2K, F-1) flat candidates of the fused scores, ties to the lower flat index.
* `beam_topk` / `install` -- a CPU stand-in for kernels.beam_topk that takes the LM keywords, installed over
                    tests/beam_emulator.py's to run BeamGraph with an LM without a GPU."""
import math

import torch

import beam_emulator


def fused_lprobs(logits, lm_logits, lm_weight, mask, inv_temp, eos, t, min_len, max_len, dtype=torch.float32):
    lp = torch.log_softmax(logits.to(dtype) * inv_temp, dim=-1)
    V_lm = lm_logits.shape[1]
    lp[:, :V_lm] += torch.log_softmax(lm_logits.to(dtype), dim=-1) * lm_weight
    if t < min_len:
        lp[:, eos] = -math.inf
    lp[lp != lp] = -math.inf
    lp = lp + mask.to(dtype)
    if t >= max_len:
        lp[:, :eos] = -math.inf
        lp[:, eos + 1:] = -math.inf
    return lp


def topk(logits, lm_logits, lm_weight, cum, mask, inv_temp, eos, t, min_len, max_len, K, dtype=torch.float32):
    """Returns (score [B, n], token [B, n], beam [B, n]), n = min(2K, F - 1)."""
    lp = fused_lprobs(logits, lm_logits, lm_weight, mask, inv_temp, eos, t, min_len, max_len, dtype)
    BK, V = lp.shape
    B = BK // K
    flat = lp.view(B, K, V)[:, 0] if t == 0 else (lp + cum.to(dtype)[:, None]).view(B, K * V)
    n = min(2 * K, flat.shape[1] - 1)
    vals, idx = torch.sort(flat, dim=1, descending=True, stable=True)
    return vals[:, :n], idx[:, :n] % V, idx[:, :n] // V


def beam_topk(logits, cum, mask, inv_temp, eos, t, min_len, max_len, cand_score, cand_token, cand_beam, *, K,
              lm_logits=None, lm_weight=0.0):
    if lm_logits is None:
        return beam_emulator.beam_topk(logits, cum, mask, inv_temp, eos, t, min_len, max_len, cand_score, cand_token,
                                       cand_beam, K=K)
    if lm_logits.shape[1] > logits.shape[1]:
        raise ValueError("the LM vocabulary is larger than the decoder's")
    cs, ct, cb = topk(logits, lm_logits, lm_weight, cum, mask, inv_temp, eos, int(t), int(min_len), int(max_len), K)
    n = cs.shape[1]
    cand_score[:, :n], cand_token[:, :n], cand_beam[:, :n] = cs, ct.to(cand_token.dtype), cb.to(cand_beam.dtype)


def install(monkeypatch):
    from speecht5_b200 import kernels as K
    beam_emulator.install(monkeypatch)
    monkeypatch.setattr(K, "beam_topk", beam_topk)


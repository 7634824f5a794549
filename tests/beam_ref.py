"""Torch statement of beam search for text output (speecht5/sequence_generator.py:207-654 with ctc_weight 0, no LM, no
prefix tokens; candidate selection fairseq/search.py:117-144), written from those semantics:

* `topk`   -- st5_beam_topk: the masked log-probabilities of every row and each sentence's best min(2K, F-1) flat
              candidates, ties to the lower flat index (any dtype: float64 for kernel checks, float32 for parity).
* `update` -- st5_beam_update on the lineage state of speecht5_b200/incremental.BeamGraph (CPU tensors, in place).
* `search` -- the whole search in the reference's own layout (tokens [B*K, max_len+2], cumulative scores
              [B*K, max_len+1], rows reordered by index_select), for a logits function of the token prefix.
"""
import math

import torch


def masked_lprobs(logits, mask, inv_temp, eos, t, min_len, max_len, dtype=torch.float32):
    lp = torch.log_softmax(logits.to(dtype) * inv_temp, dim=-1)
    if t < min_len:
        lp[:, eos] = -math.inf
    lp[lp != lp] = -math.inf
    lp = lp + mask.to(dtype)
    if t >= max_len:
        lp[:, :eos] = -math.inf
        lp[:, eos + 1:] = -math.inf
    return lp


def topk(logits, cum, mask, inv_temp, eos, t, min_len, max_len, K, dtype=torch.float32):
    """Returns (score [B, n], token [B, n], beam [B, n]), n = min(2K, F - 1)."""
    lp = masked_lprobs(logits, mask, inv_temp, eos, t, min_len, max_len, dtype)
    BK, V = lp.shape
    B = BK // K
    flat = lp.view(B, K, V)[:, 0] if t == 0 else (lp + cum.to(dtype)[:, None]).view(B, K * V)
    n = min(2 * K, flat.shape[1] - 1)
    vals, idx = torch.sort(flat, dim=1, descending=True, stable=True)
    return vals[:, :n], idx[:, :n] % V, idx[:, :n] // V


def update(st, K, V, eos, normalize, len_penalty):
    """st5_beam_update (include/speecht5_b200.h) on the state dict, one sentence at a time."""
    t, maxl = int(st["t"]), int(st["max_len"])
    T = st["lin"].shape[1]
    n = min(2 * K, (V if t == 0 else K * V) - 1)
    for s in range(st["finished"].shape[0]):
        if st["finished"][s]:
            continue
        cs, ct, cb = st["cand_score"][s, :n], st["cand_token"][s, :n], st["cand_beam"][s, :n]
        ign = st["ignore"][s * K:(s + 1) * K].clone()
        em = [bool(ct[c] == eos and cs[c] != -math.inf) and not (c < K and bool(ign[c])) for c in range(n)]
        eos_c = [c for c in range(min(n, K)) if em[c]]
        held = int(st["fin_n"][s])
        for c in eos_c[:K - held]:
            x, slot = s * K + int(cb[c]), int(st["fin_n"][s])
            lin = st["lin"][x]
            cum = [float(st["score"][int(lin[j + 1]), j + 1]) for j in range(t)] + [float(cs[c])]
            cum = torch.tensor(cum, dtype=torch.float32)
            pos = cum.clone()
            pos[1:] = cum[1:] - cum[:-1]
            st["fin_tok"][s, slot, :t + 1] = torch.tensor(
                [int(st["tok"][int(lin[j + 1]), j + 1]) for j in range(t)] + [eos], dtype=st["fin_tok"].dtype)
            st["fin_pos"][s, slot, :t + 1] = pos
            st["fin_len"][s, slot] = t + 1
            sc = cs[c].clone()
            st["fin_score"][s, slot] = sc / (t + 1) ** len_penalty if normalize else sc
            st["fin_n"][s] += 1
        if (eos_c and (int(st["fin_n"][s]) == K or t == maxl)) or t >= maxl:
            st["finished"][s] = 1
            continue
        m2 = [em[c] or (c < K and bool(ign[c])) for c in range(n)]
        order = [c for c in range(n) if not m2[c]] + [c for c in range(n) if m2[c]]
        active = order[:K]
        rows = st["lin"][s * K:(s + 1) * K, :t + 1].clone()
        for k, c in enumerate(active):
            r = s * K + k
            st["lin"][r, :t + 1] = rows[int(cb[c])]
            st["lin"][r, t + 1] = r
            st["tok"][r, t + 1] = ct[c]
            st["score"][r, t + 1] = cs[c]
            st["parent"][r] = s * K + int(cb[c])
            st["cur_tok"][r] = ct[c]
            st["cur_score"][r] = cs[c]
            st["ignore"][r] = int(m2[c])
        assert T >= t + 2
    st["stop"][t] = int(bool(st["finished"].all()))


def search(logits_fn, B, K, V, max_len, min_len=1, mask=None, inv_temp=1.0, eos=2, pad=1, normalize=True,
           len_penalty=1.0):
    """The search in the reference's layout. logits_fn(tokens [B*K, t+1]) -> logits [B*K, V] of the last position.
    Returns per sentence its hypotheses sorted by score descending (dicts as SequenceGenerator returns them)."""
    BK = B * K
    mask = torch.zeros(V) if mask is None else mask
    tokens = torch.full((BK, max_len + 2), pad, dtype=torch.long)
    tokens[:, 0] = eos
    scores = torch.zeros(BK, max_len + 1)
    ignore = torch.zeros(B, K, dtype=torch.bool)
    finalized = [[] for _ in range(B)]
    finished = [False] * B
    for t in range(max_len + 1):
        logits = logits_fn(tokens[:, :t + 1])
        cum = scores[:, t - 1] if t > 0 else torch.zeros(BK)
        cs, ct, cb = topk(logits, cum, mask, inv_temp, eos, t, min_len, max_len, K)
        n = cs.shape[1]
        em = ct.eq(eos) & cs.ne(-math.inf)
        em[:, :K][ignore] = False
        new_order = torch.arange(BK)
        for s in range(B):
            if finished[s]:
                continue
            eos_c = [c for c in range(min(n, K)) if em[s, c]]
            for c in eos_c:
                x = s * K + int(cb[s, c])
                if len(finalized[s]) < K:
                    tk = tokens[x, 1:t + 2].clone()
                    tk[t] = eos
                    pos = scores[x, :t + 1].clone()
                    pos[t] = cs[s, c]
                    pos[1:] = pos[1:] - pos[:-1]
                    sc = cs[s, c] / (t + 1) ** len_penalty if normalize else cs[s, c]
                    finalized[s].append({"tokens": tk, "score": sc, "attention": None, "alignment": torch.empty(0),
                                         "positional_scores": pos})
            if eos_c and (len(finalized[s]) == K or t == max_len):
                finished[s] = True
        if all(finished) or t == max_len:
            break
        m2 = em.clone()
        m2[:, :K] = ignore | em[:, :K]
        active_mask = m2.long() * 2 * K + torch.arange(n)
        new_ign, active = torch.topk(active_mask, k=K, dim=1, largest=False)
        ignore = new_ign.ge(2 * K)
        bb = torch.gather(cb + torch.arange(B)[:, None] * K, 1, active).view(-1)
        live = torch.tensor([not f for f in finished]).repeat_interleave(K)
        new_order = torch.where(live, bb, new_order)
        nt, nsc = torch.gather(ct, 1, active).view(-1), torch.gather(cs, 1, active).view(-1)
        tokens[:, :t + 1] = tokens[new_order, :t + 1]
        scores[:, :t] = scores[new_order, :t]
        tokens[:, t + 1] = torch.where(live, nt, tokens[:, t + 1])
        scores[:, t] = torch.where(live, nsc, scores[:, t])
    return [sorted(f, key=lambda h: -float(h["score"])) for f in finalized]

"""CPU stand-ins for kernels.beam_topk, kernels.beam_update and kernels.attn_lineage_fwd (st5_beam_topk, st5_beam_update,
st5_attn_lineage_fwd): tests install them with monkeypatch, next to tests/gemm_emulator.py, to run
T5TransformerModel.generate_text_beam's host composition (speecht5_b200/incremental.BeamGraph) without a GPU."""
import beam_ref
import decode_emulator


def attn_lineage_fwd(q, k, v, out, *, H, scale, key_pad=None, kv_rows=None, kv_div=1):
    """Gather each query row's keys / values explicitly, then the fp64 one-row attention of tests/decode_emulator."""
    import torch
    B, Tk = q.shape[0], k.shape[1]
    if kv_rows is not None:
        rows = kv_rows[:, :Tk].long()
        j = torch.arange(Tk)[None].expand(B, Tk)
        kg, vg = k[rows, j], v[rows, j]
    else:
        idx = torch.arange(B) // kv_div
        kg, vg = k[idx], v[idx]
    decode_emulator.attn_decode_fwd(q, kg, vg, out, H=H, scale=scale, key_pad=key_pad)


def beam_topk(logits, cum, mask, inv_temp, eos, t, min_len, max_len, cand_score, cand_token, cand_beam, *, K):
    cs, ct, cb = beam_ref.topk(logits, cum, mask, inv_temp, eos, int(t), int(min_len), int(max_len), K)
    n = cs.shape[1]
    cand_score[:, :n], cand_token[:, :n], cand_beam[:, :n] = cs, ct.to(cand_token.dtype), cb.to(cand_beam.dtype)


def beam_update(st, *, K, V, eos, normalize, len_penalty):
    beam_ref.update(st, K, V, eos, normalize, len_penalty)


def install(monkeypatch):
    from speecht5_b200 import kernels as K
    monkeypatch.setattr(K, "attn_lineage_fwd", attn_lineage_fwd)
    monkeypatch.setattr(K, "beam_topk", beam_topk)
    monkeypatch.setattr(K, "beam_update", beam_update)

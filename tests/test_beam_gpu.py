"""-m gpu: beam search on the device. st5_beam_topk against an fp64 statement, st5_beam_update against tests/beam_ref.py
on hand-made candidate lists, st5_attn_lineage_fwd against explicitly gathered keys (and bit-identical to
st5_attn_decode_fwd with an identity table), generate_text_beam against the reference SequenceGenerator's hypotheses
(tests/golden/ref_beam_tiny.npz) in parity mode, bf16 graph / eager / batch-1 agreement, and a full-size Base run."""
import math

import numpy as np
import pytest
import torch

import beam_ref
from test_beam_cpu import V as VOCAB, cases, check_hypos, load

pytestmark = pytest.mark.gpu
INF = float("inf")


def _scalars(dev, *v):
    return [torch.tensor([x], dtype=torch.int64, device=dev) for x in v]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("K", [1, 2, 5, 10, 16])
@pytest.mark.parametrize("V", [81, 1000, 8000, 32000])
def test_beam_topk_against_fp64(cuda, V, K, dtype):
    from speecht5_b200 import kernels
    B, eos = 3, 2
    g = torch.Generator().manual_seed(V * 31 + K)
    # logits on a 1/8 grid: many exact ties inside a row (same log-probability bit for bit), resolved by lower index
    x = (torch.randint(-32, 33, (B * K, V), generator=g).float() / 8).to(dtype)
    x[0, 5] = -INF
    x[1 % (B * K), 7:11] = -INF
    if B * K > 2:
        x[2, 3] = float("nan")  # the whole row becomes -inf, like log_softmax
    mask = torch.zeros(V)
    mask[1], mask[V - 1], mask[3] = -INF, -INF, -0.5
    cum = -torch.rand(B * K, generator=g) * 4
    for t, mn, mx in ((0, 1, 20), (3, 1, 20), (2, 5, 20), (20, 1, 20)):
        n = min(2 * K, (V if t == 0 else K * V) - 1)
        cs = torch.full((B, 2 * K), float("nan"), device=cuda)
        ct = torch.full((B, 2 * K), -7, dtype=torch.int32, device=cuda)
        cb = torch.full((B, 2 * K), -7, dtype=torch.int32, device=cuda)
        tt, mnt, mxt = _scalars(cuda, t, mn, mx)
        kernels.beam_topk(x.to(cuda), cum.to(cuda), mask.to(cuda), 1.25, eos, tt, mnt, mxt, cs, ct, cb, K=K)
        torch.cuda.synchronize()
        cs, ct, cb = cs.cpu(), ct.cpu().long(), cb.cpu().long()
        assert torch.isnan(cs[:, n:]).all() and (ct[:, n:] == -7).all() and (cb[:, n:] == -7).all()
        ws, wt, wb = beam_ref.topk(x.double(), cum.double(), mask.double(), 1.25, eos, t, mn, mx, K, dtype=torch.float64)
        lp = beam_ref.masked_lprobs(x.double(), mask.double(), 1.25, eos, t, mn, mx, torch.float64)
        if t > 0:
            lp = lp + cum.double()[:, None]
        for s in range(B):
            got = cs[s, :n].double()
            assert ((got[:-1] >= got[1:]) | torch.isinf(got[1:])).all()
            fin = torch.isfinite(ws[s])
            assert torch.equal(torch.isfinite(got), fin), (t, s)
            assert torch.allclose(got[fin], ws[s][fin], rtol=1e-5, atol=1e-4), (t, s)
            # each chosen (beam, token) has the score of its rank; where the fp64 ranks are well separated, it IS the rank's
            at = lp[s * K + cb[s, :n], ct[s, :n]]
            assert torch.allclose(at[fin], ws[s][fin], rtol=1e-5, atol=1e-4)
            gap = torch.cat([torch.tensor([INF]), (ws[s][:-1] - ws[s][1:]).abs(), torch.tensor([INF])])
            sep = (gap[:-1] > 1e-3) & (gap[1:] > 1e-3) | ~fin
            assert torch.equal(ct[s, :n][sep], wt[s][sep]) and torch.equal(cb[s, :n][sep], wb[s][sep]), (t, s)
            # exact ties inside one row: lower token first
            for i in range(n - 1):
                if cb[s, i] == cb[s, i + 1] and cs[s, i] == cs[s, i + 1]:
                    assert ct[s, i] < ct[s, i + 1]
            assert len({(int(b), int(k)) for b, k in zip(cb[s, :n], ct[s, :n])}) == n
            if t == 0:
                assert (cb[s, :n] == 0).all()


def _state(B, K, T, dev="cpu"):
    i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
    return dict(t=torch.zeros(1, dtype=torch.int64, device=dev), max_len=torch.zeros(1, dtype=torch.int64, device=dev),
                cand_score=torch.zeros((B, 2 * K), **f32), cand_token=torch.zeros((B, 2 * K), **i32),
                cand_beam=torch.zeros((B, 2 * K), **i32), lin=torch.zeros((B * K, T), **i32),
                tok=torch.zeros((B * K, T), **i32), score=torch.zeros((B * K, T), **f32),
                ignore=torch.zeros(B * K, **i32), finished=torch.zeros(B, **i32), parent=torch.zeros(B * K, **i32),
                cur_tok=torch.zeros(B * K, dtype=torch.int64, device=dev), cur_score=torch.zeros(B * K, **f32),
                fin_n=torch.zeros(B, **i32), fin_tok=torch.zeros((B, K, T), **i32),
                fin_pos=torch.zeros((B, K, T), **f32), fin_len=torch.zeros((B, K), **i32),
                fin_score=torch.zeros((B, K), **f32), stop=torch.zeros(T, **i32))


def _random_history(st, K, t, g):
    """A consistent lineage state after t steps: random parents per step, tokens >= 4, decreasing cumulative scores."""
    BK = st["lin"].shape[0]
    st["lin"][:, 0] = torch.arange(BK, dtype=torch.int32)
    for j in range(t):
        for r in range(BK):
            s = r // K
            p = s * K + int(torch.randint(0, K, (1,), generator=g))
            st["lin"][r, :j + 1] = st["lin"][p, :j + 1].clone() if j > 0 else p
        st["lin"][:, j + 1] = torch.arange(BK, dtype=torch.int32)
        st["tok"][:, j + 1] = torch.randint(4, 50, (BK,), generator=g, dtype=torch.int32)
        st["score"][:, j + 1] = st["score"][st["lin"][:, j].long(), j] - torch.rand(BK, generator=g)
    st["cur_score"] = st["score"][torch.arange(BK), t].clone()


CASES = {
    # name: (K, t, max_len, eos candidate positions, ignore positions, finalized already, normalize, len_penalty)
    "eos_inside_top_k": (4, 5, 20, [1], [], 0, True, 1.0),
    "eos_outside_top_k": (4, 5, 20, [5, 6], [], 0, True, 1.0),
    "list_reaches_k": (3, 6, 20, [0, 2], [], 2, True, 1.0),
    "cands_to_ignore_nonempty": (3, 4, 20, [0, 1, 3, 4, 5], [], 0, True, 1.0),
    "ignored_positions_skip_eos": (4, 5, 20, [0, 2], [0, 2], 1, True, 1.0),
    "t_equals_max_len": (4, 8, 8, [0, 1, 2, 3], [], 0, True, 1.0),
    "minus_inf_eos": (4, 5, 20, [1, 2], [], 0, True, 1.0),
    "len_penalty_not_one": (4, 5, 20, [0, 3], [], 0, True, 0.6),
    "normalize_off": (4, 5, 20, [0, 3], [], 0, False, 1.0),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_beam_update_against_beam_ref(cuda, name):
    from speecht5_b200 import kernels
    K, t, maxl, eos_pos, ign, held, normalize, lpen = CASES[name]
    B, T, V, eos = 3, 32, 60, 2
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    st = _state(B, K, T)
    _random_history(st, K, t, g)
    st["t"][0], st["max_len"][0] = t, maxl
    st["finished"][2] = 1  # a finished sentence is left alone
    for s in range(B):
        sc = torch.sort(st["cur_score"][s * K:(s + 1) * K].max() - torch.rand(2 * K, generator=g) * 3, descending=True)[0]
        st["cand_score"][s] = sc
        st["cand_token"][s] = torch.randint(4, V, (2 * K,), generator=g, dtype=torch.int32)
        st["cand_beam"][s] = torch.randint(0, K, (2 * K,), generator=g, dtype=torch.int32)
        for c in eos_pos:
            st["cand_token"][s, c] = eos
        if name == "minus_inf_eos":
            st["cand_score"][s, 2:] = -INF
        for c in ign:
            st["ignore"][s * K + c] = 1
        st["fin_n"][s] = held
    want = {k: v.clone() for k, v in st.items()}
    beam_ref.update(want, K, V, eos, normalize, lpen)
    got = {k: v.to(cuda) for k, v in st.items()}
    kernels.beam_update(got, K=K, V=V, eos=eos, normalize=normalize, len_penalty=lpen)
    torch.cuda.synchronize()
    for k in want:
        if k in ("fin_pos", "fin_score"):
            assert torch.allclose(got[k].cpu(), want[k], rtol=1e-6, atol=1e-6), (name, k)
        else:
            assert torch.equal(got[k].cpu(), want[k]), (name, k)
    # the cases do what their names say
    if name == "list_reaches_k" or name == "t_equals_max_len":
        assert want["finished"][:2].all()
    if name == "cands_to_ignore_nonempty":
        assert want["ignore"][:2 * K].any()


def test_lineage_attention_against_explicit_gather(cuda):
    from speecht5_b200 import kernels
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float32, torch.bfloat16):
        for span in (7, 64, 65, 200):
            B, K, H = 2, 3, 2
            BK, T = B * K, span + 5
            q = torch.randn(BK, 1, H * 64, generator=g).to(dtype)
            kv = torch.randn(BK, T, 2 * H * 64, generator=g).to(dtype)
            rows = torch.randint(0, BK, (BK, T), generator=g, dtype=torch.int32)
            pad = (torch.rand(BK, span, generator=g) < 0.2).to(torch.uint8)
            pad[:, 0] = 0
            qd, kvd, rd, pd = q.to(cuda), kv.to(cuda), rows.to(cuda), pad.to(cuda)
            out = torch.empty(BK, 1, H * 64, dtype=dtype, device=cuda)
            kernels.attn_lineage_fwd(qd, kvd[:, :span, :H * 64], kvd[:, :span, H * 64:], out, H=H, scale=0.125,
                                     key_pad=pd, kv_rows=rd)
            j = torch.arange(span)[None].expand(BK, span)
            kg, vg = kv[rows[:, :span].long(), j, :H * 64].double(), kv[rows[:, :span].long(), j, H * 64:].double()
            s = torch.einsum("bhc,bjhc->bhj", q[:, 0].double().reshape(BK, H, 64), kg.reshape(BK, span, H, 64)) * 0.125
            p = torch.softmax(s.masked_fill(pad.bool()[:, None], -INF), -1)
            ref = torch.einsum("bhj,bjhc->bhc", p, vg.reshape(BK, span, H, 64)).reshape(BK, 1, H * 64)
            tol = 1e-5 if dtype == torch.float32 else 2e-2
            assert (out.cpu().double() - ref).abs().max() < tol, (dtype, span)
            # kv_div: K query rows share one key / value row
            enc = kv[:B].to(cuda)
            out2 = torch.empty_like(out)
            kernels.attn_lineage_fwd(qd, enc[:, :span, :H * 64], enc[:, :span, H * 64:], out2, H=H, scale=0.125,
                                     key_pad=pd, kv_div=K)
            out3 = torch.empty_like(out)
            encK = enc.repeat_interleave(K, 0)
            kernels.attn_decode_fwd(qd, encK[:, :span, :H * 64], encK[:, :span, H * 64:], out3, H=H, scale=0.125,
                                    key_pad=pd)
            assert torch.equal(out2, out3), (dtype, span)
            # identity table, kv_div 1: bit-identical to st5_attn_decode_fwd
            ident = torch.arange(BK, dtype=torch.int32, device=cuda)[:, None].expand(BK, T).contiguous()
            kernels.attn_lineage_fwd(qd, kvd[:, :span, :H * 64], kvd[:, :span, H * 64:], out2, H=H, scale=0.125,
                                     key_pad=pd, kv_rows=ident)
            kernels.attn_decode_fwd(qd, kvd[:, :span, :H * 64], kvd[:, :span, H * 64:], out3, H=H, scale=0.125,
                                    key_pad=pd)
            assert torch.equal(out2, out3), (dtype, span)


def _fixture_model(cuda, dtype, blob):
    from test_ref_pin_gpu import TINY_CONV, _build
    from helpers import NO_DROPOUT, TINY
    over = dict(TINY, **NO_DROPOUT, bert_init=True, build_speech_encoder=True, build_text_decoder=True,
                conv_feature_layers=TINY_CONV, feature_grad_mult=1.0, conv_pos=16, conv_pos_groups=4, use_conv_pos=True,
                use_sinc_pos=True, mask_prob=0.0, mask_channel_prob=0.0, max_text_positions=600)
    m = _build(cuda, dtype, **over)
    m.load_state_dict({k[6:]: torch.from_numpy(v) for k, v in blob.items() if k.startswith("state/")}, strict=False)
    return m.eval()


MASK_KW = dict(blank=VOCAB - 1, mask_idx=VOCAB - 2)


def test_generate_text_beam_against_the_reference_generator(cuda):
    blob = load()
    m = _fixture_model(cuda, torch.float32, blob)
    source, pm = torch.from_numpy(blob["in/source"]).to(cuda), torch.from_numpy(blob["in/padding_mask"]).to(cuda)
    for mode in (True, "graph", "graph"):  # (the second graph call replays the captured graphs)
        for ci, K, mn, mx, lp in cases(blob):
            got = m.generate_text_beam(source, pm, beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp,
                                       use_cache=mode, **MASK_KW)
            for b, hs in enumerate(got):
                for i, h in enumerate(hs):
                    n = int(blob[f"c{ci}/len"][b, i])
                    assert h["tokens"].tolist() == blob[f"c{ci}/tokens"][b, i, :n].tolist(), (mode, ci, b, i)
                    assert abs(float(h["score"]) - float(blob[f"c{ci}/score"][b, i])) < 2e-3, (mode, ci, b, i)
                    want = torch.from_numpy(blob[f"c{ci}/pos"][b, i, :n]).double()
                    err = (h["positional_scores"].cpu().double() - want).abs()
                    assert (err <= 1e-3 * want.abs().clamp_min(1.0) + 1e-3 * float(want.cumsum(0).abs().max())).all()


def test_bf16_graph_eager_batch1_and_beam1(cuda):
    from speecht5_b200.generator import BeamSearchGenerator, GreedyGenerator
    from types import SimpleNamespace
    blob = load()
    m = _fixture_model(cuda, torch.bfloat16, blob)
    source, pm = torch.from_numpy(blob["in/source"]).to(cuda), torch.from_numpy(blob["in/padding_mask"]).to(cuda)
    kw = dict(beam_size=5, max_len_b=16, **MASK_KW)
    eager = m.generate_text_beam(source, pm, use_cache=True, **kw)
    graph = m.generate_text_beam(source, pm, use_cache="graph", **kw)
    for e, g in zip(eager, graph):
        assert [h["tokens"].tolist() for h in e] == [h["tokens"].tolist() for h in g]
        assert len(e) == 5
    for b in range(source.shape[0]):
        one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], use_cache="graph", **kw)[0]
        assert [h["tokens"].tolist() for h in one] == [h["tokens"].tolist() for h in graph[b]]
    vocab = SimpleNamespace(pad=lambda: 1, eos=lambda: 2, unk=lambda: 3)
    sample = {"net_input": {"source": source, "padding_mask": pm}}
    b1 = BeamSearchGenerator([m], vocab, beam_size=1, max_len_b=16, use_cache="graph", **MASK_KW).generate([m], sample)
    gg = GreedyGenerator([m], vocab, max_len_b=16, use_cache="graph", **MASK_KW).generate([m], sample)
    assert [h[0]["tokens"].tolist() for h in b1] == [h[0]["tokens"].tolist() for h in gg]


def test_full_size_base_beam5_graph(cuda):
    from test_ref_pin_gpu import _build
    m = _build(cuda, torch.bfloat16, build_speech_encoder=True, build_text_decoder=True, bert_init=True,
               encoder_layerdrop=0.0, decoder_layerdrop=0.0, max_text_positions=600).eval()
    g = torch.Generator().manual_seed(0)
    wav = (torch.randn(8, 160000, generator=g) * 0.1).to(cuda)
    pm = torch.zeros(8, 160000, dtype=torch.bool, device=cuda)
    kw = dict(beam_size=5, max_len_b=40, min_len=1)
    graph = m.generate_text_beam(wav, pm, use_cache="graph", **kw)
    eager = m.generate_text_beam(wav, pm, use_cache=True, **kw)
    for e, gr in zip(eager, graph):
        assert len(gr) == 5
        sc = [float(h["score"]) for h in gr]
        assert sc == sorted(sc, reverse=True) and all(math.isfinite(x) for x in sc)
        assert [h["tokens"].tolist() for h in e] == [h["tokens"].tolist() for h in gr]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_hypotheses_past_130_tokens_graph_eager_and_batch1(cuda, dtype):
    """min_len 132 of max_len 160 on the fixture model: the graph's buffers and position table well past the fixture's
    16 steps (bucket 256). Graph and eager agree bit for bit; each sentence alone gives its row of the batch."""
    blob = load()
    m = _fixture_model(cuda, dtype, blob)
    source, pm = torch.from_numpy(blob["in/source"]).to(cuda), torch.from_numpy(blob["in/padding_mask"]).to(cuda)
    kw = dict(beam_size=4, max_len_b=160, min_len=132, **MASK_KW)
    graph = m.generate_text_beam(source, pm, use_cache="graph", **kw)
    eager = m.generate_text_beam(source, pm, use_cache=True, **kw)
    for e, g in zip(eager, graph):
        assert len(g) == 4 and all(len(h["tokens"]) > 130 for h in g)
        assert [h["tokens"].tolist() for h in e] == [h["tokens"].tolist() for h in g]
        assert [float(h["score"]) for h in e] == [float(h["score"]) for h in g]
        assert all(torch.equal(a["positional_scores"], b["positional_scores"]) for a, b in zip(e, g))
    for b in range(source.shape[0]):
        one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], use_cache="graph", **kw)[0]
        assert [h["tokens"].tolist() for h in one] == [h["tokens"].tolist() for h in graph[b]], b

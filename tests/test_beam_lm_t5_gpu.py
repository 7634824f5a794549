"""-m gpu: LM shallow fusion with SpeechT5's own LM architecture (`transformer_lm_t5`: heads of 80 channels) on the
device. generate_text_beam(lm=...) against the reference SequenceGenerator's hypotheses with a tiny transformer_lm_t5
fused in (tests/golden/ref_beam_lm_t5_tiny.npz) in parity mode and bf16, eager and graph, each sentence alone against
its batch row, through BeamSearchGenerator and build_generator; the LM's forward against the reference's probe; and a
full-size run: a random-weight 20 x 1280 transformer_lm_t5 with the Base ASR model, beam 5, 8 utterances (graph against
eager, the LM moving the search), and the cached step's log-probabilities against an fp64 restatement of fairseq's
transformer_lm on the same weights."""
import gc
import math
from argparse import Namespace
from types import SimpleNamespace

import pytest
import torch

from test_beam_cpu import load as load_asr
from test_beam_gpu import MASK_KW, _fixture_model
from test_beam_lm_gpu import _check_close
from test_beam_lm_t5_cpu import build_lm, cases, fake_fairseq_lm, load

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_graphs():
    """Collect the captured graphs when each test ends; and leave torch's global CPU generator as the test found it (the
    tests seed it for their random LMs; none draws from the device generator), so that the tests after these draw what
    they would without them."""
    state = torch.get_rng_state()
    yield
    gc.collect()
    torch.cuda.empty_cache()
    torch.set_rng_state(state)


def test_lm_forward_against_the_reference_probe(cuda):
    from speecht5_b200.ops import RT
    blob = load()
    RT.dtype = torch.float32
    RT.invalidate_shadows()
    lm = build_lm(blob).to(cuda)
    got = lm.log_probs(torch.from_numpy(blob["probe/tokens"]).to(cuda)).cpu()
    want = torch.from_numpy(blob["probe/lprobs"])
    assert torch.allclose(got, want, rtol=0, atol=2e-3), float((got - want).abs().max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fixture_graph_eager_and_batch1(cuda, dtype):
    """Parity mode (fp32) reproduces the reference's hypotheses, scores and positional scores eager, in graph form and
    sentence by sentence. bf16 is held to the same hypotheses where its rounding stays inside the fixture's 1e-3
    candidate gaps, which it need not (as for the 64-wide LM): there the LM must move the search, every hypothesis list
    must be sorted and finite, and graph / eager / batch-1 must agree."""
    blob, asr = load(), load_asr()
    m = _fixture_model(cuda, dtype, asr)
    lm = build_lm(blob).to(cuda)
    source, pm = torch.from_numpy(asr["in/source"]).to(cuda), torch.from_numpy(asr["in/padding_mask"]).to(cuda)
    moved = False
    for ci, K, mn, mx, lp, w in cases(blob):
        kw = dict(beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, lm=lm, lm_weight=w, **MASK_KW)
        eager = m.generate_text_beam(source, pm, use_cache=True, **kw)
        graph = m.generate_text_beam(source, pm, use_cache="graph", **kw)
        again = m.generate_text_beam(source, pm, use_cache="graph", **kw)
        if dtype == torch.float32:
            for got in (eager, graph, again):
                _check_close(got, blob, ci, 2e-3)
        else:
            plain = m.generate_text_beam(source, pm, use_cache="graph",
                                         **{k: v for k, v in kw.items() if k not in ("lm", "lm_weight")})
            moved |= any([h["tokens"].tolist() for h in a] != [h["tokens"].tolist() for h in b]
                         for a, b in zip(graph, plain))
            for hs in graph:
                sc = [float(h["score"]) for h in hs]
                assert len(hs) == K and sc == sorted(sc, reverse=True) and all(math.isfinite(x) for x in sc)
        for e, g in zip(graph, again):
            assert [h["tokens"].tolist() for h in e] == [h["tokens"].tolist() for h in g]
        for e, g in zip(eager, graph):
            assert [h["tokens"].tolist() for h in e] == [h["tokens"].tolist() for h in g]
            assert [float(h["score"]) for h in e] == [float(h["score"]) for h in g]
            assert all(torch.equal(a["positional_scores"], b["positional_scores"]) for a, b in zip(e, g))
        for b in range(source.shape[0]):
            one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], use_cache="graph", **kw)[0]
            assert [h["tokens"].tolist() for h in one] == [h["tokens"].tolist() for h in graph[b]], (ci, b)
            if dtype == torch.float32:
                _check_close([one], {k: (v[b:b + 1] if k.startswith(f"c{ci}/") and v.ndim >= 2 else v)
                                     for k, v in blob.items()}, ci, 2e-3)
    if dtype == torch.bfloat16:
        assert moved


def test_generators_with_the_t5_lm(cuda):
    from speecht5_b200.generator import BeamSearchGenerator
    from speecht5_b200.tasks.speecht5 import SpeechT5Task
    from test_beam_cpu import V
    blob, asr = load(), load_asr()
    m = _fixture_model(cuda, torch.float32, asr)
    fs = fake_fairseq_lm(blob).to(cuda)
    source, pm = torch.from_numpy(asr["in/source"]).to(cuda), torch.from_numpy(asr["in/padding_mask"]).to(cuda)
    sample = {"net_input": {"source": source, "padding_mask": pm}}
    vocab = SimpleNamespace(pad=lambda: 1, eos=lambda: 2, unk=lambda: 3)
    for ci in (0, 2, 3):
        _, K, mn, mx, lp, w = list(cases(blob))[ci]
        gen = BeamSearchGenerator([m], vocab, beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, lm_model=fs,
                                  lm_weight=w, use_cache="graph", **MASK_KW)
        _check_close(gen.generate([m], sample), blob, ci, 2e-3)
    task = SpeechT5Task.__new__(SpeechT5Task)
    task.args, task.dicts = SimpleNamespace(ctc_weight=0.0), {"text": vocab}
    task.blank_symbol_idx, task.mask_idx = V - 1, V - 2
    _, K, mn, mx, lp, w = list(cases(blob))[2]
    args = SimpleNamespace(beam=K, max_len_a=0, max_len_b=mx, min_len=mn, unnormalized=False, lenpen=lp, unkpen=0.0)
    g = task.build_generator([m], args, seq_gen_cls=BeamSearchGenerator,
                             extra_gen_cls_kwargs={"lm_model": fs, "lm_weight": w})
    _check_close(task.inference_step(g, [m], sample), blob, 2, 2e-3)


# ============================================================================================ full size
def _random_t5_lm(V_lm, dev):
    """transformer_lm_t5 at its own sizes with random weights scaled so activations stay O(1): Linear and embedding
    weights N(0, 1 / fan_in), biases N(0, 0.02^2), LayerNorms N(1, 0.1^2) / N(0, 0.1^2)."""
    from speecht5_b200.lm import TransformerLM
    torch.manual_seed(0)
    lm = TransformerLM(Namespace(arch="transformer_lm_t5"), V_lm)
    with torch.no_grad():
        for name, p in lm.named_parameters():
            if "layer_norm" in name:
                p.normal_(1.0 if name.endswith("weight") else 0.0, 0.1)
            elif name.endswith("bias"):
                p.normal_(0.0, 0.02)
            else:
                p.normal_(0.0, p.shape[1] ** -0.5)
    return lm.to(dev)


def fairseq_lm_fp64(lm, tokens):
    """fairseq's transformer_lm forward (TransformerDecoder without encoder attention, pre-LN layers, fairseq's
    MultiheadAttention with q scaled by head_dim^-0.5 before q.k, GELU (erf), final LayerNorm, untied output
    projection) restated in fp64 on the LM's weights -> log-probabilities [B, T, V_lm]."""
    from speecht5_b200.lm import fairseq_sinusoid_table_fp32
    F = torch.nn.functional
    d = lm.decoder
    W = {k: v.detach().double() for k, v in lm.state_dict().items()}
    C, H = lm.args.decoder_embed_dim, lm.args.decoder_attention_heads
    hd = C // H
    B, T = tokens.shape
    pe = fairseq_sinusoid_table_fp32(lm.padding_idx + 1 + T, C, lm.padding_idx)[lm.padding_idx + 1:].double()
    x = lm.embed_scale * W["decoder.embed_tokens.weight"][tokens] + pe.to(tokens.device)[None]
    causal = torch.full((T, T), -math.inf, dtype=torch.float64, device=tokens.device).triu(1)

    def ln(x, p):
        return F.layer_norm(x, (C,), W[p + ".weight"], W[p + ".bias"], 1e-5)

    def lin(x, p):
        return F.linear(x, W[p + ".weight"], W.get(p + ".bias"))
    for i in range(len(d.layers)):
        p = f"decoder.layers.{i}."
        h = ln(x, p + "self_attn_layer_norm")
        q = lin(h, p + "self_attn.q_proj") * hd ** -0.5
        k, v = lin(h, p + "self_attn.k_proj"), lin(h, p + "self_attn.v_proj")
        q, k, v = (t.view(B, T, H, hd).transpose(1, 2) for t in (q, k, v))
        a = torch.softmax(q @ k.transpose(-1, -2) + causal, -1) @ v
        x = x + lin(a.transpose(1, 2).reshape(B, T, C), p + "self_attn.out_proj")
        h = ln(x, p + "final_layer_norm")
        x = x + lin(F.gelu(lin(h, p + "fc1")), p + "fc2")
    x = ln(x, "decoder.layer_norm")
    return torch.log_softmax(F.linear(x, W["decoder.output_projection.weight"]), -1)


def test_full_size_t5_lm_cached_step_against_fp64(cuda):
    """The LM half of BeamGraph's step body (embedding + position of the newest token, decoder_step over a static
    lineage-read cache with the pad mask of positions not yet written, the output projection) at its full size in bf16,
    one position per step for 12 steps, against fairseq_lm_fp64 on the same weights.

    Bound: every layer rounds to bf16 (unit 2^-9 relative, round to nearest) the inputs of its GEMMs and attention --
    the LayerNorm outputs, q | k | v and the cache, the attention output, the FFN hidden -- and its two residual sums,
    and its six weight matrices are read as bf16 copies of the fp32 weights the restatement uses: about twelve
    roundings per layer, 240 over the 20 layers and a few more at the ends, of errors independent in sign, so the hidden
    state's relative error grows like a random walk, sqrt(256) 2^-9 ~ 3.1 %. A logit is a 1280-term dot product of that
    state with an output row, so its error is ~3.1 % of the logits' rms scale, and a log-probability (logit minus
    log-sum-exp) at most twice that. The test takes four times this estimate:
    |lp - lp_64| <= 8 sqrt(256) 2^-9 rms(logits of the row) = 0.25 rms, a quarter of the row's spread.
    """
    from speecht5_b200 import ops
    from speecht5_b200.incremental import _StaticCache, decoder_step
    from speecht5_b200.ops import RT
    RT.dtype = torch.bfloat16
    RT.invalidate_shadows()
    V_lm, BK, T, rows = 79, 6, 12, 64
    lm = _random_t5_lm(V_lm, cuda)
    g = torch.Generator().manual_seed(1)
    tokens = torch.randint(4, V_lm, (BK, T), generator=g)
    tokens[:, 0] = 2
    tokens = tokens.to(cuda)
    C = lm.args.decoder_embed_dim
    with torch.no_grad():
        cache = _StaticCache([], [torch.zeros((BK, rows, 2 * C), dtype=RT.dtype, device=cuda)
                                  for _ in lm.decoder.layers], None, rows)
        emb, pe = lm.scaled_embedding(), torch.zeros((rows, C), device=cuda)
        pe[:T + 1] = lm.positions(T + 1, cuda)
        lin = torch.arange(BK, dtype=torch.int32, device=cuda)[:, None].expand(BK, rows).contiguous()
        pos = torch.arange(rows, device=cuda)
        got = []
        for t in range(T):
            t_dev = torch.tensor([t], device=cuda)
            y = ops.scaled_posenc(pe.index_select(0, t_dev), lm._unit, 0.0, tokens=tokens[:, t:t + 1].contiguous(),
                                  emb=emb, padding_idx=lm.padding_idx)
            self_pad = (pos > t_dev).to(torch.uint8)[None].expand(BK, rows).contiguous()
            z, _ = decoder_step(lm.decoder, y, cache, t_dev=t_dev, span=rows, self_pad=self_pad, self_rows=lin)
            got.append(torch.log_softmax(lm.output_layer(z)[:, -1].float(), -1))
        got = torch.stack(got, 1).double()
        want = fairseq_lm_fp64(lm, tokens)
        logits_rms = (want - want.mean(-1, keepdim=True)).pow(2).mean(-1, keepdim=True).sqrt()
    bound = 8 * math.sqrt(256) * 2.0 ** -9 * logits_rms
    ratio = float(((got - want).abs() / bound).max())
    print(f"\nfull-size transformer_lm_t5 cached step: max |lp - lp_64| / bound = {ratio:.3g} "
          f"(max err {float((got - want).abs().max()):.3g}, rms logits {float(logits_rms.mean()):.3g})")
    assert ratio <= 1.0
    # the bound separates: the same comparison one position off fails it
    assert float(((got[:, 1:] - want[:, :-1]).abs() / bound[:, 1:]).max()) > 1.0


def test_full_size_base_with_t5_lm_graph_and_eager(cuda):
    from speecht5_b200.lm import TransformerLM
    from test_ref_pin_gpu import _build
    m = _build(cuda, torch.bfloat16, build_speech_encoder=True, build_text_decoder=True, bert_init=True,
               encoder_layerdrop=0.0, decoder_layerdrop=0.0, max_text_positions=600).eval()
    V = m.text_decoder_postnet.output_projection.weight.shape[0]
    # (every parameter N(0, 0.05^2), as the 64-wide full-size test draws its LM: with an untrained ASR model the fused
    # scores are near-flat, and an LM this gentle moves the search without making near-ties of bf16 rounding size)
    torch.manual_seed(0)
    lm = TransformerLM(Namespace(arch="transformer_lm_t5"), V - 2)
    for p in lm.parameters():
        torch.nn.init.normal_(p, std=0.05)
    lm = lm.to(cuda)
    g = torch.Generator().manual_seed(0)
    wav = (torch.randn(8, 160000, generator=g) * 0.1).to(cuda)
    pm = torch.zeros(8, 160000, dtype=torch.bool, device=cuda)
    kw = dict(beam_size=5, max_len_b=40, min_len=1, lm=lm, lm_weight=0.5)
    graph = m.generate_text_beam(wav, pm, use_cache="graph", **kw)
    eager = m.generate_text_beam(wav, pm, use_cache=True, **kw)
    plain = m.generate_text_beam(wav, pm, use_cache="graph", beam_size=5, max_len_b=40, min_len=1)
    assert any([h["tokens"].tolist() for h in a] != [h["tokens"].tolist() for h in b] for a, b in zip(graph, plain))
    # Graph and eager replay the same kernels, but at this size not bit for bit (as in the 64-wide full-size test), and
    # an untrained ASR model leaves many candidates tied to bf16 rounding: each rank must hold the same hypothesis, or
    # two whose scores agree to that rounding (a near-tie swapped), and every rank's score must agree.
    same = 0
    for e, gr in zip(eager, graph):
        assert len(gr) == len(e) == 5
        sc = [float(h["score"]) for h in gr]
        assert sc == sorted(sc, reverse=True) and all(math.isfinite(x) for x in sc)
        assert all(abs(float(h["score"]) - x) <= 1e-3 * abs(x) + 1e-3 for h, x in zip(e, sc))
        same += sum(a["tokens"].tolist() == b["tokens"].tolist() for a, b in zip(e, gr))
    assert same >= 0.9 * 8 * 5, same

"""LM shallow fusion for text beam search (lm.TransformerLM, generate_text_beam(lm=...), the generators' lm_model /
lm_weight) without a GPU: the reference SequenceGenerator's own hypotheses with fairseq's transformer_lm fused in
(tests/golden/ref_beam_lm_tiny.npz, make_golden_beam_lm.py) reproduced by the host composition (incremental.BeamGraph)
on emulated kernels; the LM against the reference LM's log-probabilities; the constructors, the options that raise, and
the fp64 statement of the fused score (tests/beam_lm_ref.py)."""
import math
import os
import re
import shutil
import subprocess
import sys
from argparse import Namespace
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import beam_lm_ref
import beam_ref
from test_beam_cpu import MASK_KW, V, check_hypos, model, src  # noqa: F401  (model: the fixture of the ASR model)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
N_CASES = 5


def load():
    return dict(np.load(os.path.join(GOLD, "ref_beam_lm_tiny.npz")))


def lm_args(blob):
    L, C, H, F, tps = (int(x) for x in blob["lm_args"])
    return Namespace(decoder_layers=L, decoder_embed_dim=C, decoder_attention_heads=H, decoder_ffn_embed_dim=F,
                     tokens_per_sample=tps, activation_fn="relu")


def lm_state(blob):
    return {k[3:]: torch.from_numpy(v) for k, v in blob.items() if k.startswith("lm/")}


def build_lm(blob):
    from speecht5_b200.lm import TransformerLM
    lm = TransformerLM(lm_args(blob), V - 2)
    lm.load_fairseq_state(lm_state(blob))
    return lm


def fake_fairseq_lm(blob):
    """What generate.py hands over as lm_model: a module with .args and .decoder under fairseq's names, plus fairseq's
    bookkeeping buffers."""
    inner = build_lm(blob)
    m = torch.nn.Module()
    m.decoder = inner.decoder
    m.decoder.register_buffer("version", torch.tensor([3.0]))
    m.decoder.adaptive_softmax = None
    m.args = lm_args(blob)
    return m


def cases(blob):
    for ci in range(N_CASES):
        K, mn, mx = (int(x) for x in blob[f"c{ci}/meta"])
        yield ci, K, mn, mx, float(blob[f"c{ci}/len_penalty"]), float(blob[f"c{ci}/lm_weight"])


@pytest.fixture
def fused(model, monkeypatch):  # noqa: F811
    beam_lm_ref.install(monkeypatch)
    m, _ = model
    yield m, build_lm(load()), load()


def test_fixture_is_what_the_reference_produces_now():
    from oracle import ref_loader as rl
    if not rl.available():
        pytest.skip("reference tree not available")
    sys.path.insert(0, GOLD)
    import make_golden_beam_lm as mg
    fresh, blob = mg.make(), load()
    assert sorted(fresh) == sorted(blob)
    for k in blob:
        assert np.array_equal(fresh[k], blob[k]), k


def test_lm_matches_the_reference_log_probabilities(fused):
    _, lm, blob = fused
    tok = torch.from_numpy(blob["probe/tokens"])
    got = lm.log_probs(tok)
    want = torch.from_numpy(blob["probe/lprobs"])
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=0, atol=2e-4), float((got - want).abs().max())


def test_from_fairseq_and_load_lm_round_trip(fused, tmp_path):
    from speecht5_b200.lm import TransformerLM, load_lm
    _, lm, blob = fused
    want = lm.state_dict()

    def same(other):
        got = other.state_dict()
        assert sorted(got) == sorted(want)
        for k in want:
            assert torch.equal(got[k], want[k]), k
    fs = fake_fairseq_lm(blob)
    same(TransformerLM.from_fairseq(fs))
    assert TransformerLM.from_fairseq(lm) is lm
    state = dict(fs.state_dict(), **{"decoder.embed_positions._float_tensor": torch.zeros(1)})
    torch.save({"model": state, "args": lm_args(blob)}, tmp_path / "args.pt")
    torch.save({"model": state, "cfg": {"model": vars(lm_args(blob))}}, tmp_path / "cfg.pt")
    same(load_lm(str(tmp_path / "args.pt")))
    same(load_lm(str(tmp_path / "cfg.pt")))
    with pytest.raises(ValueError):
        torch.save({"model": state}, tmp_path / "none.pt")
        load_lm(str(tmp_path / "none.pt"))
    # tied output projection: the checkpoint holds the embedding only
    tied = Namespace(**vars(lm_args(blob)), share_decoder_input_output_embed=True)
    t = TransformerLM(tied, V - 2)
    t.load_fairseq_state({k: v for k, v in lm_state(blob).items() if k != "decoder.output_projection.weight"})
    assert t.decoder.output_projection.weight is t.decoder.embed_tokens.weight


@pytest.mark.parametrize("opt", [dict(adaptive_input=True), dict(adaptive_softmax_cutoff="10,20"),
                                 dict(tie_adaptive_weights=True), dict(character_embeddings=True),
                                 dict(layernorm_embedding=True), dict(decoder_input_dim=32), dict(decoder_output_dim=32),
                                 dict(cross_self_attention=True), dict(quant_noise_pq=0.1), dict(quant_noise_scalar=0.1),
                                 dict(no_token_positional_embeddings=True), dict(decoder_attention_heads=2),
                                 dict(activation_fn="tanh")])
def test_unbuilt_options_raise(opt):
    from speecht5_b200.lm import TransformerLM
    args = Namespace(decoder_layers=1, decoder_embed_dim=64, decoder_attention_heads=1, decoder_ffn_embed_dim=128)
    for k, v in opt.items():
        setattr(args, k, v)
    with pytest.raises(NotImplementedError):
        TransformerLM(args, 10)


def test_lm_options_built(fused):
    """learned positions, no_scale_embedding, gelu, no final norm: forward against a plain torch statement."""
    from speecht5_b200.lm import TransformerLM
    torch.manual_seed(3)
    args = Namespace(decoder_layers=1, decoder_embed_dim=64, decoder_attention_heads=1, decoder_ffn_embed_dim=96,
                     decoder_learned_pos=True, max_target_positions=12, no_scale_embedding=True, activation_fn="gelu",
                     no_decoder_final_norm=True)
    lm = TransformerLM(args, 20)
    for p in lm.parameters():
        torch.nn.init.normal_(p, std=0.2)
    assert lm.decoder.layer_norm is None and lm.embed_scale == 1.0
    tok = torch.tensor([[2, 5, 7, 9, 4]])
    d, x = lm.decoder, None
    x = d.embed_tokens.weight[tok] + d.embed_positions.weight[2:7][None]
    for layer in d.layers:
        h = torch.nn.functional.layer_norm(x, (64,), layer.self_attn_layer_norm.weight, layer.self_attn_layer_norm.bias)
        sa = layer.self_attn
        q, k, v = (torch.nn.functional.linear(h, p.weight, p.bias) for p in (sa.q_proj, sa.k_proj, sa.v_proj))
        s = (q * sa.scaling) @ k.transpose(1, 2) + torch.triu(torch.full((5, 5), -math.inf), 1)
        x = x + torch.nn.functional.linear(torch.softmax(s, -1) @ v, sa.out_proj.weight, sa.out_proj.bias)
        h = torch.nn.functional.layer_norm(x, (64,), layer.final_layer_norm.weight, layer.final_layer_norm.bias)
        x = x + layer.fc2(torch.nn.functional.gelu(layer.fc1(h)))
    want = torch.log_softmax(x @ d.output_projection.weight.t(), -1)
    assert torch.allclose(lm.log_probs(tok), want, atol=1e-4)
    with pytest.raises(NotImplementedError, match="learned LM positions"):
        lm.positions(13, "cpu")  # (12 positions: max_target_positions)


def test_generate_text_beam_with_lm_matches_the_reference(fused):
    m, lm, blob = fused
    source, pm = src(dict(np.load(os.path.join(GOLD, "ref_beam_tiny.npz"))))
    for ci, K, mn, mx, lp, w in cases(blob):
        got = m.generate_text_beam(source, pm, beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, use_cache=True,
                                   lm=lm, lm_weight=w, **MASK_KW)
        check_hypos(got, blob, ci)
    # each sentence alone gives its own hypotheses
    ci, K, mn, mx, lp, w = list(cases(blob))[2]
    for b in range(source.shape[0]):
        one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp,
                                   lm=lm, lm_weight=w, **MASK_KW)
        check_hypos(one, blob, ci, rows=[b])


def test_generators_and_build_generator_with_lm(fused):
    from speecht5_b200.generator import BeamSearchGenerator, GreedyGenerator
    from speecht5_b200.tasks.speecht5 import SpeechT5Task
    m, _, blob = fused
    source, pm = src(dict(np.load(os.path.join(GOLD, "ref_beam_tiny.npz"))))
    sample = {"net_input": {"source": source, "padding_mask": pm}}
    vocab = SimpleNamespace(pad=lambda: 1, eos=lambda: 2, unk=lambda: 3)
    fs = fake_fairseq_lm(blob)
    _, K, mn, mx, lp, w = list(cases(blob))[2]
    gen = BeamSearchGenerator([m], vocab, beam_size=K, max_len_b=mx, lm_model=fs, lm_weight=w, **MASK_KW)
    check_hypos(gen.generate([m], sample), blob, 2)
    task = SpeechT5Task.__new__(SpeechT5Task)
    task.args, task.dicts = SimpleNamespace(ctc_weight=0.0), {"text": vocab}
    task.blank_symbol_idx, task.mask_idx = V - 1, V - 2
    # beam 1 with an LM: the reference's beam search with K = 1, through the default generator class too
    _, K0, _, mx0, _, w0 = list(cases(blob))[0]
    assert K0 == 1
    for cls in (None, BeamSearchGenerator):
        args = SimpleNamespace(beam=1, max_len_a=0, max_len_b=mx0, min_len=1, unnormalized=False, lenpen=1.0, unkpen=0.0)
        g = task.build_generator([m], args, seq_gen_cls=cls, extra_gen_cls_kwargs={"lm_model": fs, "lm_weight": w0})
        check_hypos(task.inference_step(g, [m], sample), blob, 0)
    args = SimpleNamespace(beam=K, max_len_a=0, max_len_b=mx, min_len=1, unnormalized=False, lenpen=1.0, unkpen=0.0)
    g = task.build_generator([m], args, seq_gen_cls=BeamSearchGenerator,
                             extra_gen_cls_kwargs={"lm_model": fs, "lm_weight": w})
    check_hypos(task.inference_step(g, [m], sample), blob, 2)
    with pytest.raises(NotImplementedError):
        task.inference_step(g, [m], sample, prefix_tokens=torch.zeros(4, 1, dtype=torch.long))
    with pytest.raises(NotImplementedError):
        BeamSearchGenerator([m], vocab, beam_size=5, ctc_weight=0.3, lm_model=fs)
    with pytest.raises(NotImplementedError):
        GreedyGenerator([m], vocab, ctc_weight=0.3, lm_model=fs)


def test_lm_vocabulary_larger_than_the_decoders_raises(fused):
    from speecht5_b200.lm import TransformerLM
    m, _, blob = fused
    source, pm = src(dict(np.load(os.path.join(GOLD, "ref_beam_tiny.npz"))))
    big = TransformerLM(lm_args(blob), V + 1)
    with pytest.raises(ValueError, match="larger"):
        m.generate_text_beam(source, pm, beam_size=2, max_len_b=4, lm=big, **MASK_KW)
    with pytest.raises(TypeError):
        m.generate_text_beam(source, pm, beam_size=2, max_len_b=4, lm=fake_fairseq_lm(blob), **MASK_KW)


def test_fused_score_statement():
    """beam_lm_ref.fused_lprobs in float64 against the formula written out per element, and its corner cases."""
    g = torch.Generator().manual_seed(7)
    BK, Vd, V_lm, T = 4, 11, 9, 0.7
    x = torch.randn(BK, Vd, generator=g, dtype=torch.float64) * 3
    y = torch.randn(BK, V_lm, generator=g, dtype=torch.float64) * 3
    mask = torch.zeros(Vd, dtype=torch.float64)
    mask[1] = -math.inf
    mask[3] = -0.5
    got = beam_lm_ref.fused_lprobs(x, y, 0.4, mask, 1 / T, 2, 5, 1, 10, torch.float64)
    for r in range(BK):
        lse_x = math.log(sum(math.exp(float(x[r, u]) / T) for u in range(Vd)))
        lse_y = math.log(sum(math.exp(float(y[r, u])) for u in range(V_lm)))
        for v in range(Vd):
            want = float(x[r, v]) / T - lse_x + (0.4 * (float(y[r, v]) - lse_y) if v < V_lm else 0.0) + float(mask[v])
            assert abs(float(got[r, v]) - want) <= 1e-12 or (math.isinf(want) and got[r, v] == want), (r, v)
    # weight 0 with finite LM logits: the plain masked log-probabilities, bit for bit
    plain = beam_ref.masked_lprobs(x, mask, 1 / T, 2, 0, 1, 10, torch.float64)
    assert torch.equal(beam_lm_ref.fused_lprobs(x, y, 0.0, mask, 1 / T, 2, 0, 1, 10, torch.float64), plain)
    # NaN handling after the add: weight 0 against an LM log-probability of -inf, and a NaN LM row, give -inf
    y2 = y.clone()
    y2[0, 4] = -math.inf
    y2[1, 0] = math.nan
    z = beam_lm_ref.fused_lprobs(x, y2, 0.0, mask, 1 / T, 2, 3, 1, 10, torch.float64)
    assert z[0, 4] == -math.inf and torch.isfinite(z[0, 5])
    assert (z[1, :V_lm] == -math.inf).all() and torch.isfinite(z[1, V_lm:]).all()
    # max_len: only eos survives; min_len: eos is banned
    assert (beam_lm_ref.fused_lprobs(x, y, 0.4, mask, 1, 2, 10, 1, 10, torch.float64)[:, [0, 1, 3, 4]] == -math.inf).all()
    assert (beam_lm_ref.fused_lprobs(x, y, 0.4, mask, 1, 2, 0, 1, 10, torch.float64)[:, 2] == -math.inf).all()


def test_lm_row_kernels_fit_their_launch_bounds_without_spills():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("cuobjdump or library not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    seen = set()
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res):
        name, regs, stack, local = m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))
        if "lm_fused_row_topk" in name:
            assert stack == 0 and local == 0 and regs * 256 <= 65536, (name, regs, stack, local)
            seen.add(name)
    assert len(seen) == 2, sorted(seen)  # (fp32 and bf16 decoder logits)

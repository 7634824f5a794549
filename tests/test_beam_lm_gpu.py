"""-m gpu: LM shallow fusion on the device. st5_beam_topk_lm against the fp64 statement of tests/beam_lm_ref.py (fp32 /
bf16 operands, row pitches past V and V_lm, NaN sentinels in either operand), bit-identical to st5_beam_topk at
lm_weight 0, its argument errors; generate_text_beam(lm=...) against the reference SequenceGenerator's hypotheses with
fairseq's transformer_lm fused in (tests/golden/ref_beam_lm_tiny.npz) in parity mode and bf16, eager and graph, graph
and eager bit for bit, each sentence alone against its batch row; a full-size Base ASR + base transformer_lm run."""
import ctypes as C
import gc
import math

import pytest
import torch

import beam_lm_ref
from test_beam_cpu import load as load_asr
from test_beam_gpu import MASK_KW, _fixture_model
from test_beam_lm_cpu import build_lm, cases, load

pytestmark = pytest.mark.gpu
INF = float("inf")


@pytest.fixture(autouse=True)
def _release_graphs():
    """The captured graphs (and their private memory pools) live on the models in a reference cycle: collect them when
    each test ends rather than at some later collection."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _scalars(dev, *v):
    return [torch.tensor([x], dtype=torch.int64, device=dev) for x in v]


def _pitched(rows, cols, pad, dtype, g, scale, dev):
    """[rows, cols] values in a [rows, cols + pad] buffer whose tail columns are NaN (read past the row = NaN result)."""
    buf = torch.full((rows, cols + pad), float("nan"))
    buf[:, :cols] = torch.randn(rows, cols, generator=g) * scale
    return buf.to(dtype).to(dev)[:, :cols]


def _run(kernels, x, y, w, cum, mask, t, mn, mx, K, dev, eos=2):
    B = x.shape[0] // K
    cs = torch.full((B, 2 * K), float("nan"), device=dev)
    ct = torch.full((B, 2 * K), -7, dtype=torch.int32, device=dev)
    cb = torch.full((B, 2 * K), -7, dtype=torch.int32, device=dev)
    tt, mnt, mxt = _scalars(dev, t, mn, mx)
    kw = {} if y is None else dict(lm_logits=y, lm_weight=w)
    kernels.beam_topk(x, cum, mask, 1.25, eos, tt, mnt, mxt, cs, ct, cb, K=K, **kw)
    torch.cuda.synchronize()
    return cs.cpu(), ct.cpu().long(), cb.cpu().long()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("K", [1, 2, 5, 16])
@pytest.mark.parametrize("V", [3, 81, 8000, 32768])
@pytest.mark.parametrize("lm_v", ["1", "V-2", "V"])
def test_topk_lm_against_fp64(cuda, V, K, dtype, lm_v):
    from speecht5_b200 import kernels
    V_lm = {"1": 1, "V-2": max(1, V - 2), "V": V}[lm_v]
    B, eos, w = 2, 2, 0.6
    g = torch.Generator().manual_seed(V * 131 + K * 7 + V_lm)
    x = _pitched(B * K, V, 5, dtype, g, 3.0, cuda)
    y = _pitched(B * K, V_lm, 3, dtype, g, 3.0, cuda)
    if B * K > 2:
        x[1, 0] = float("nan")   # the decoder row -> -inf everywhere
        y[2, 0] = float("nan")   # the LM row -> -inf on v < V_lm only
    mask = torch.zeros(V, device=cuda)
    mask[1 % V] = -INF
    cum = (-torch.rand(B * K, generator=g) * 4).to(cuda)
    for t, mn, mx in ((0, 1, 20), (3, 1, 20), (2, 5, 20), (20, 1, 20)):
        n = min(2 * K, (V if t == 0 else K * V) - 1)
        cs, ct, cb = _run(kernels, x, y, w, cum, mask, t, mn, mx, K, cuda)
        assert torch.isnan(cs[:, n:]).all() and (ct[:, n:] == -7).all() and (cb[:, n:] == -7).all()
        lp = beam_lm_ref.fused_lprobs(x.double().cpu(), y.double().cpu(), w, mask.double().cpu(), 1.25, eos, t, mn, mx,
                                      torch.float64)
        if t > 0:
            lp = lp + cum.double().cpu()[:, None]
        ws, wt, wb = beam_lm_ref.topk(x.double().cpu(), y.double().cpu(), w, cum.double().cpu(), mask.double().cpu(),
                                      1.25, eos, t, mn, mx, K, dtype=torch.float64)
        for s in range(B):
            got = cs[s, :n].double()
            assert ((got[:-1] >= got[1:]) | torch.isinf(got[1:])).all(), (t, s)
            fin = torch.isfinite(ws[s])
            assert torch.equal(torch.isfinite(got), fin), (t, s)
            tol = 1e-5 * ws[s][fin].abs() + 2e-4
            assert ((got[fin] - ws[s][fin]).abs() <= tol).all(), (t, s)
            at = lp[s * K + cb[s, :n], ct[s, :n]]  # each chosen (beam, token) carries its own fp64 score
            assert ((at[fin] - got[fin]).abs() <= tol).all(), (t, s)
            assert len({(int(b), int(k)) for b, k in zip(cb[s, :n], ct[s, :n])}) == n
            gap = torch.cat([torch.tensor([INF]), (ws[s][:-1] - ws[s][1:]).abs(), torch.tensor([INF])])
            sep = (gap[:-1] > 1e-3) & (gap[1:] > 1e-3) | ~fin
            assert torch.equal(ct[s, :n][sep], wt[s][sep]) and torch.equal(cb[s, :n][sep], wb[s][sep]), (t, s)
            if t == 0:
                assert (cb[s, :n] == 0).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_weight_zero_is_beam_topk_bit_for_bit(cuda, dtype):
    from speecht5_b200 import kernels
    g = torch.Generator().manual_seed(5)
    for K, V in ((1, 81), (5, 8000), (16, 32768)):
        x = _pitched(2 * K, V, 4, dtype, g, 3.0, cuda)
        y = _pitched(2 * K, V - 2, 7, dtype, g, 3.0, cuda)
        mask = torch.zeros(V, device=cuda)
        mask[1] = -INF
        cum = (-torch.rand(2 * K, generator=g) * 4).to(cuda)
        for t in (0, 3):
            a = _run(kernels, x, y, 0.0, cum, mask, t, 1, 20, K, cuda)
            b = _run(kernels, x, None, 0.0, cum, mask, t, 1, 20, K, cuda)
            assert all(torch.equal(p, q) for p, q in zip(a[1:], b[1:]))
            assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))


def test_argument_errors(cuda):
    from speecht5_b200 import _lib, kernels
    lib = _lib.load()
    one = C.c_void_p(16)

    def call(V_lm, lm_ld, lm=one, V=81):
        return lib.st5_beam_topk_lm(one, V, 0, 1, 2, V, one, one, 1.0, 2, one, one, one, one, one, one, one, lm, lm_ld,
                                    0, V_lm, 0.5, None)
    assert call(0, 81) == -2 and b"st5_beam_topk_lm" in lib.st5_last_error()
    assert call(82, 82) == -2 and call(81, 80) == -6 and call(79, 78) == -6 and call(79, 79, lm=None) == -3
    assert call(79, 79, V=40000) == -2
    x = torch.zeros(2, 81, device=cuda)
    s, i32 = torch.zeros(1, 4, device=cuda), torch.zeros(1, 4, dtype=torch.int32, device=cuda)
    tt, = _scalars(cuda, 0)
    with pytest.raises(ValueError, match="larger"):
        kernels.beam_topk(x, x[:, 0].contiguous(), x[0].contiguous(), 1.0, 2, tt, tt, tt, s, i32, i32.clone(), K=2,
                          lm_logits=torch.zeros(2, 82, device=cuda), lm_weight=0.5)


def _lm(cuda, blob):
    return build_lm(blob).to(cuda)


def _check_close(got, blob, ci, tol):
    for b, hs in enumerate(got):
        for i, h in enumerate(hs):
            n = int(blob[f"c{ci}/len"][b, i])
            assert h["tokens"].tolist() == blob[f"c{ci}/tokens"][b, i, :n].tolist(), (ci, b, i)
            assert abs(float(h["score"]) - float(blob[f"c{ci}/score"][b, i])) < tol, (ci, b, i)
            want = torch.from_numpy(blob[f"c{ci}/pos"][b, i, :n]).double()
            err = (h["positional_scores"].cpu().double() - want).abs()
            assert (err <= tol * want.abs().clamp_min(1.0) + tol * float(want.cumsum(0).abs().max())).all(), (ci, b, i)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fixture_graph_eager_and_batch1(cuda, dtype):
    """Parity mode (fp32) reproduces the reference's hypotheses in eager and graph form. bf16 is not pinned to them:
    its rounding exceeds the fixture's 1e-3 candidate gaps (sentence 3 of case 2 takes another path after 6 tokens);
    there the LM must still move the search, and graph / eager / batch-1 must agree."""
    blob, asr = load(), load_asr()
    m = _fixture_model(cuda, dtype, asr)
    lm = _lm(cuda, blob)
    source, pm = torch.from_numpy(asr["in/source"]).to(cuda), torch.from_numpy(asr["in/padding_mask"]).to(cuda)
    moved = False
    for ci, K, mn, mx, lp, w in cases(blob):
        kw = dict(beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, lm=lm, lm_weight=w, **MASK_KW)
        eager = m.generate_text_beam(source, pm, use_cache=True, **kw)
        graph = m.generate_text_beam(source, pm, use_cache="graph", **kw)
        again = m.generate_text_beam(source, pm, use_cache="graph", **kw)  # (replays the captured graphs)
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
        if ci == 2:
            for b in range(source.shape[0]):
                one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], use_cache="graph", **kw)[0]
                assert [h["tokens"].tolist() for h in one] == [h["tokens"].tolist() for h in graph[b]], b
    if dtype == torch.bfloat16:
        assert moved


def test_generators_with_fairseq_style_lm(cuda):
    from types import SimpleNamespace
    from speecht5_b200.generator import BeamSearchGenerator
    from test_beam_lm_cpu import fake_fairseq_lm
    blob, asr = load(), load_asr()
    m = _fixture_model(cuda, torch.float32, asr)
    fs = fake_fairseq_lm(blob).to(cuda)
    source, pm = torch.from_numpy(asr["in/source"]).to(cuda), torch.from_numpy(asr["in/padding_mask"]).to(cuda)
    vocab = SimpleNamespace(pad=lambda: 1, eos=lambda: 2, unk=lambda: 3)
    for ci in (0, 2):
        _, K, mn, mx, lp, w = list(cases(blob))[ci]
        gen = BeamSearchGenerator([m], vocab, beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, lm_model=fs,
                                  lm_weight=w, use_cache="graph", **MASK_KW)
        _check_close(gen.generate([m], {"net_input": {"source": source, "padding_mask": pm}}), blob, ci, 2e-3)


def test_full_size_base_with_base_lm_graph_and_eager(cuda):
    from argparse import Namespace
    from speecht5_b200.lm import TransformerLM
    from test_ref_pin_gpu import _build
    m = _build(cuda, torch.bfloat16, build_speech_encoder=True, build_text_decoder=True, bert_init=True,
               encoder_layerdrop=0.0, decoder_layerdrop=0.0, max_text_positions=600).eval()
    V = m.text_decoder_postnet.output_projection.weight.shape[0]
    torch.manual_seed(0)
    lm = TransformerLM(Namespace(decoder_layers=6, decoder_embed_dim=512, decoder_attention_heads=8,
                                 decoder_ffn_embed_dim=2048), V - 2)
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
    for e, gr in zip(eager, graph):
        assert len(gr) == 5
        sc = [float(h["score"]) for h in gr]
        assert sc == sorted(sc, reverse=True) and all(math.isfinite(x) for x in sc)
        assert [h["tokens"].tolist() for h in e] == [h["tokens"].tolist() for h in gr]
        # (same hypotheses; at this size graph and eager scores agree to bf16 rounding, not bit for bit)
        assert all(abs(float(h["score"]) - x) <= 1e-3 * abs(x) + 1e-3 for h, x in zip(e, sc))

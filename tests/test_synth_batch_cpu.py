"""Batched speech synthesis (generate_speech_batch) without a GPU: the batched step body of incremental.SynthesisGraph,
run eagerly on emulated kernels, gives every utterance of a TTS and a VC batch what the reference's own batch-1
generate_speech gives it (tests/golden/ref_synth_batch_tiny.npz, tests/golden/make_golden_synth_batch.py) and what this
project's generate_speech gives it alone, and keeps the reference's stopping rule (models/speecht5.py:1222-1245) per
utterance; ops.attention_decode's views and the one-row dispatch of ops.attention against a torch statement."""
import os
import sys

import numpy as np
import pytest
import torch

import decode_emulator
from helpers import NO_DROPOUT, rel
from test_vc_cpu import _emulated, load_generation_state, mv, vc_case

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_synth_batch as ms  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402

needs_ref = pytest.mark.skipif(not rl.available(), reason="reference tree not available")


def synth_fixture():
    return dict(np.load(os.path.join(HERE, "golden", "ref_synth_batch_tiny.npz")))


def synth_model(dev):
    """The product model with the fixture's weights (filled from the parameter names), eval mode, no update."""
    _, model, _, _ = vc_case(dev)
    return model.eval()


def batch_inputs(blob, batch, dev):
    t = lambda k: torch.from_numpy(blob[f"in/{batch}/{k}"]).to(dev)  # noqa: E731
    if batch == "tts":
        return dict(src_tokens=t("tokens"), src_lengths=t("lengths").cpu(), spkembs=t("spkembs"))
    return dict(source=t("source"), padding_mask=t("padding_mask"), spkembs=t("spkembs"))


def alone_kwargs(inp, b):
    """generate_speech inputs of utterance b of a batch, padding stripped."""
    if "src_tokens" in inp:
        n = int(inp["src_lengths"][b])
        return dict(src_tokens=inp["src_tokens"][b:b + 1, :n], spkembs=inp["spkembs"][b:b + 1])
    n = int((~inp["padding_mask"][b]).sum())
    return dict(source=inp["source"][b:b + 1, :n], padding_mask=inp["padding_mask"][b:b + 1, :n],
                spkembs=inp["spkembs"][b:b + 1])


def check_against_fixture(model, blob, dev, bound, mode):
    """Every utterance of both batches, every case: length exact, mel / stop probabilities / attention within `bound`
    of the reference; each also equals this project's batch-1 generate_speech in the same mode within 1e-6."""
    bias = model.speech_decoder_postnet.prob_out.bias
    for case, (kw, offsets) in ms.CASES.items():
        for batch in ("tts", "vc"):
            inp = batch_inputs(blob, batch, dev)
            with torch.no_grad():
                bias.add_(offsets[batch])
            got = model.generate_speech_batch(**inp, attention=True, use_cache=mode, **kw)
            for b, res in enumerate(got):
                for g, k in zip(res, ("mel", "probs", "attn")):
                    want = torch.from_numpy(blob[f"{batch}/{case}/{b}/{k}"])
                    assert g.shape == want.shape, (batch, case, b, k, g.shape, want.shape)
                    assert rel(g, want) < bound, (batch, case, b, k, rel(g, want))
                alone = model.generate_speech(**alone_kwargs(inp, b), use_cache=mode, **kw)
                for g, a in zip(res, alone):
                    assert g.shape == a.shape and rel(g, a) < 1e-6, (batch, case, b, rel(g, a))
            with torch.no_grad():
                bias.sub_(offsets[batch])


@needs_ref
def test_committed_fixture_is_what_the_reference_produces_now():
    fresh = ms.main(path=None)
    stored = synth_fixture()
    assert set(fresh) == set(stored)
    for k in stored:
        assert np.array_equal(fresh[k], stored[k]), k


def test_fixture_covers_every_stopping_rule():
    """Between them the utterances stop on a probability, at their own maxlen, and later than a probability because
    `threshold` was passed; the ragged batches have members of different lengths in every case."""
    blob = synth_fixture()
    for batch, n in (("tts", 4), ("vc", 3)):
        lens = {case: [blob[f"{batch}/{case}/{b}/probs"].size // 2 for b in range(n)] for case in ms.CASES}
        first = {case: [(lambda h: h[0] + 1 if len(h) else None)(np.nonzero(
            (blob[f"{batch}/{case}/{b}/probs"].reshape(-1, 2) >= (0.9 if case == "threshold" else 0.5)).any(1))[0])
            for b in range(n)] for case in ms.CASES}
        assert all(len(set(v)) > 1 for v in lens.values()), (batch, lens)
        assert all(f is None for f in first["default"])  # every one at its own maxlen
        assert any(f == L for f, L in zip(first["stop"], lens["stop"]))  # a probability stop ...
        assert any(f is None for f in first["stop"])  # ... next to a maxlen stop in the same batch
        assert any(f is not None and f < L for f, L in zip(first["threshold"], lens["threshold"]))  # delayed


def test_batches_reproduce_the_reference_on_emulated_kernels(monkeypatch):
    """Within 1e-4, the bound of the batch-1 product pins on emulated kernels (tests/test_vc_cpu.py): the emulated GEMMs
    round differently from the reference's fp32 ones, and 90 autoregressive steps carry that to ~1e-5."""
    RT = _emulated(monkeypatch)
    model = synth_model(torch.device("cpu"))
    check_against_fixture(model, synth_fixture(), torch.device("cpu"), 1e-4, "graph_body_eager")
    RT.clear_static()
    RT.invalidate_shadows()


def test_attention_decode_views_and_one_row_dispatch(monkeypatch):
    """ops.attention_decode hands the kernel the q / k / v column blocks of fused projection buffers and a [B, H, 1, Tk]
    probability buffer; incremental._attend sends one-row, no-grad queries there (not to the row kernels). Checked with
    the kernel replaced by its torch statement (tests/decode_emulator.py) against softmax attention in fp64."""
    from speecht5_b200 import incremental, ops
    calls = decode_emulator.install(monkeypatch)
    g = torch.Generator().manual_seed(0)
    B, H, Tk, d = 3, 2, 70, 128
    qkv = torch.randn(B, 1, 3 * d, generator=g)
    kv = torch.randn(B, Tk, 2 * d, generator=g)
    pad = torch.zeros(B, Tk, dtype=torch.bool)
    pad[1, 20:] = True
    pad[2, 1:] = True
    with torch.no_grad():
        out, probs = incremental._attend(qkv, kv, H=H, d=d, q_col=0, k_col=0, v_col=1, scale=0.3, key_pad=pad,
                                         return_probs=True)
        self_out, none = incremental._attend(qkv, None, H=H, d=d, q_col=0, k_col=1, v_col=2, scale=0.3)
    assert len(calls) == 2 and none is None
    qh = qkv[:, 0, :d].double().reshape(B, H, 64)
    s = torch.einsum("bhc,bjhc->bhj", qh, kv[..., :d].double().reshape(B, Tk, H, 64)) * 0.3
    p = torch.softmax(s.masked_fill(pad[:, None], float("-inf")), -1)
    want = torch.einsum("bhj,bjhc->bhc", p, kv[..., d:].double().reshape(B, Tk, H, 64)).reshape(B, 1, d)
    assert out.shape == (B, 1, d) and probs.shape == (B, H, 1, Tk)
    assert rel(out, want) < 1e-6 and (probs[:, :, 0].double() - p).abs().max() < 1e-6
    v1 = qkv[:, :, 2 * d:].double().reshape(B, H, 64)
    assert rel(self_out, v1.reshape(B, 1, d)) < 1e-6  # (one key: its value)
    assert not ops.RT.attn_decode_rows  # (outside _attend, ops.attention dispatches as before)


def _vc_model(monkeypatch):
    RT = _emulated(monkeypatch)
    blob, model, _, _ = vc_case(torch.device("cpu"))
    model.eval()
    load_generation_state(model, blob)
    return RT, blob, model


def _vc_batch(blob):
    t = lambda k: torch.from_numpy(blob["batch/in/" + k])  # noqa: E731
    return t("source"), t("padding_mask"), t("spkembs")


def test_speech_encoder_on_the_padded_batch_misses_the_fixture(monkeypatch):
    """Why the encoders run per utterance: the first conv layer's GroupNorm normalises over all time steps, padding
    included, so the shortest source encoded inside the padded batch differs from the same source alone."""
    RT, blob, model = _vc_model(monkeypatch)
    source, pm, _ = _vc_batch(blob)
    n = int((~pm[2]).sum())
    with torch.no_grad():
        alone = model.forward_encoder(source[2:3, :n], padding_mask=pm[2:3, :n])["encoder_out"][0]
        padded = model.forward_encoder(source, padding_mask=pm)["encoder_out"][0][: alone.shape[0], 2:3]
    assert rel(padded, alone) > 1e-2
    RT.clear_static()
    RT.invalidate_shadows()


def _tts(monkeypatch):
    from oracle import speecht5_oracle as OT
    from speecht5_b200.models import make_args
    from speecht5_b200.models.speecht5 import T5TransformerModel
    RT = _emulated(monkeypatch)
    torch.manual_seed(3)
    over = dict(encoder_layers=2, decoder_layers=2, bert_init=True, **NO_DROPOUT)
    oracle = OT.T5TransformerModelOracle(OT.base_args(**over)).eval()
    with torch.no_grad():
        oracle.speech_decoder_postnet.prob_out.bias.fill_(-2.0)
    tts = T5TransformerModel.build_model(make_args("t5_transformer_base_asr", **over)).eval()
    tts.load_state_dict(oracle.state_dict())
    return RT, tts


def test_tts_batch_of_one_and_of_three_equal_generate_speech(monkeypatch):
    """Texts of 7 / 4 / 11 tokens with their own x-vectors through the task's collated t2s net_input (padded tokens,
    src_lengths): every utterance equals generate_speech on its own text; a batch of one returns exactly that."""
    from speecht5_b200.tasks import SpeechT5Task
    RT, tts = _tts(monkeypatch)
    g = torch.Generator().manual_seed(5)
    lens = [7, 4, 11]
    toks = torch.ones(3, max(lens), dtype=torch.long)
    for b, n in enumerate(lens):
        toks[b, :n] = torch.randint(4, 81, (n,), generator=g)
    spk = torch.randn(3, 512, generator=g)
    net_input = dict(src_tokens=toks, src_lengths=torch.tensor(lens), spkembs=spk, prev_output_tokens=None)
    got = SpeechT5Task.generate_speech_batch(None, [tts], net_input, threshold=0.9, use_cache="graph_body_eager")
    for b, n in enumerate(lens):
        alone = tts.generate_speech(src_tokens=toks[b:b + 1, :n], spkembs=spk[b:b + 1], threshold=0.9,
                                    use_cache="graph_body_eager")
        assert got[b][2] is None
        for x, y in zip(got[b][:2], alone[:2]):
            assert x.shape == y.shape and rel(x, y) < 1e-6, (b, rel(x, y))
        one = tts.generate_speech_batch(src_tokens=toks[b:b + 1, :n], spkembs=spk[b:b + 1], threshold=0.9,
                                        attention=True, use_cache="graph_body_eager")
        assert len(one) == 1
        for x, y in zip(one[0], alone):
            assert torch.equal(x, y)
    RT.clear_static()
    RT.invalidate_shadows()


def reference_stop(probs, threshold, minlen, maxlen):
    """models/speecht5.py:1222-1245 restated on a precomputed stop-probability sequence [steps, r]: the number of
    decoder steps the reference's loop runs."""
    idx = 0
    while True:
        idx += 1
        if bool((probs[idx - 1] >= threshold).any()) or idx >= maxlen:
            if idx < minlen:
                continue
            return idx


# (per row: step at which a probability first reaches the threshold or None, minlen, maxlen); threshold 0.5
STOP_TABLE = [
    [(3, 0, 10), (None, 0, 6), (5, 0, 4)],       # probability stop, own maxlen, maxlen before the probability
    [(2, 6, 12), (None, 9, 5), (1, 0, 1)],       # delayed by minlen, minlen past maxlen (clamped), stop at once
    [(None, 0, 0), (7, 7, 7), (4, 8, 20)],       # empty budget (one step), all rules at one step, minlen past a stop
]


@pytest.mark.parametrize("rows", STOP_TABLE)
def test_stop_rules_follow_the_reference_loop_per_utterance(monkeypatch, rows):
    """Synthetic stop-probability sequences replace prob_out's: the device done flags / lengths of the batched step
    equal the host restatement of the reference's loop for every row, with the reference's minlen clamp."""
    from speecht5_b200.incremental import synthesis_graph
    RT, tts = _tts(monkeypatch)
    B, steps, r = len(rows), 40, tts.reduction_factor
    seq = torch.full((steps, B, r), 0.1)
    for b, (hit, _, _) in enumerate(rows):
        if hit is not None:
            seq[hit - 1:, b, r - 1] = 0.9  # the last frame of the group reaches the threshold from step `hit` on
    sg = synthesis_graph(tts, 16, max(max(m, 1) for _, _, m in rows), "cpu", capture=False, B=B, attention=False)
    post = tts.speech_decoder_postnet
    orig = post.project

    def project(z):
        before, _ = orig(z)
        return before, torch.logit(seq[int(sg.t)])
    monkeypatch.setattr(post, "project", project)
    encs = [tts.forward_text_encoder(torch.randint(4, 81, (1, 5 + b))) for b in range(B)]
    res = sg.synthesize(encs, None, 0.5, [mn for _, mn, _ in rows], [mx for _, _, mx in rows])
    for b, (_, mn, mx) in enumerate(rows):
        want = reference_stop(seq[:, b], 0.5, min(mn, max(mx, 1)), mx)
        assert res[b][1].numel() == want * r, (rows[b], res[b][1].numel() // r, want)
        assert torch.allclose(res[b][1], seq[:want, b].reshape(-1), atol=1e-6)
    RT.clear_static()
    RT.invalidate_shadows()

"""-m gpu: batched speech synthesis on the H100 -- the split-KV decode kernel (st5_attn_decode_fwd) against fp64 torch,
its row independence, and generate_speech_batch against batch-1 generate_speech and the reference's own synthesis."""
import pytest
import torch

from helpers import rel
from test_synth_batch_cpu import check_against_fixture, synth_fixture, synth_model

pytestmark = pytest.mark.gpu
H = 12


def _inputs(B, Tk, dtype, cuda, seed=0):
    g = torch.Generator(device=cuda).manual_seed(seed)
    q = torch.randn(B, 1, 3 * H * 64, device=cuda, generator=g).to(dtype)       # q in column block 0 of a q|k|v row
    kv = torch.randn(B, Tk + 3, 2 * H * 64, device=cuda, generator=g).to(dtype)  # strided K | V, 3 spare key rows
    return q, kv[:, :Tk]


def _want(q, kv, n, scale):
    """fp64 torch: softmax(scale q k^T) v over the first n[b] keys of each utterance -> (out [B, H*64], p [B, H, Tk])."""
    B, Tk = kv.shape[0], kv.shape[1]
    qh = q[:, 0, : H * 64].double().reshape(B, H, 64)
    k = kv[..., : H * 64].double().reshape(B, Tk, H, 64)
    v = kv[..., H * 64:].double().reshape(B, Tk, H, 64)
    s = torch.einsum("bhc,bjhc->bhj", qh, k) * scale
    s = s.masked_fill(torch.arange(Tk, device=q.device)[None, None] >= n[:, None, None], float("-inf"))
    p = torch.softmax(s, -1)
    return torch.einsum("bhj,bjhc->bhc", p, v).reshape(B, H * 64), p


def _decode(q, kv, n=None, return_probs=False):
    """ops.attention_decode over the first n[b] keys of each utterance (the rest masked)."""
    from speecht5_b200 import ops
    kp = None if n is None else (torch.arange(kv.shape[1], device=q.device)[None] >= n[:, None]).to(torch.uint8)
    return ops.attention_decode(q, kv, H=H, d=H * 64, q_col=0, k_col=0, v_col=1, scale=0.125, key_pad=kp,
                                return_probs=return_probs)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B", [1, 3, 32])
@pytest.mark.parametrize("Tk", [1, 63, 64, 65, 1500])
def test_decode_kernel_against_fp64(cuda, dtype, B, Tk):
    """Per-utterance key counts from a key mask (a one-key utterance at every B, a full one at B > 1), with and without
    the returned probabilities, on the single-launch (Tk <= 64) and the split path; fp32 math on fp32 or bf16 K / V."""
    q, kv = _inputs(B, Tk, dtype, cuda)
    n = torch.randint(1, Tk + 1, (B,), device=cuda)
    n[-1] = Tk
    n[0] = 1
    want, p = _want(q, kv, n, 0.125)
    tol = 2e-6 if dtype == torch.float32 else 1e-2
    out, none = _decode(q, kv, n)
    assert none is None and rel(out[:, 0], want) < tol
    out_p, probs = _decode(q, kv, n, return_probs=True)
    assert torch.equal(out_p, out) and probs.shape == (B, H, 1, Tk)
    assert (probs[:, :, 0] - p).abs().max().item() < (1e-6 if dtype == torch.float32 else 1e-5)
    full, _ = _decode(q, kv)  # no mask: every key
    want_full, _ = _want(q, kv, torch.full((B,), Tk, device=cuda), 0.125)
    assert rel(full[:, 0], want_full) < tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_decode_rows_are_independent_of_batch_and_key_span(cuda, dtype):
    """An utterance's output and probabilities are bit-identical alone and inside a batch of 32, and in a buffer that
    holds only its valid keys (one launch when <= 64 keys) or 1 500 of which the tail is masked (split path)."""
    q, kv = _inputs(32, 1500, dtype, cuda, seed=1)
    n = torch.randint(1, 1501, (32,), device=cuda)
    n[5], n[9] = 1, 40
    full, pf = _decode(q, kv, n, return_probs=True)
    for b in (0, 5, 9, 31):
        nb = int(n[b])
        alone, pa = _decode(q[b:b + 1], kv[b:b + 1], n[b:b + 1], return_probs=True)
        narrow, pn = _decode(q[b:b + 1], kv[b:b + 1, :nb], return_probs=True)
        assert torch.equal(alone[0], full[b]) and torch.equal(narrow[0], full[b]), b
        assert torch.equal(pa[0], pf[b]) and torch.equal(pn[0, ..., :nb], pf[b, ..., :nb]), b


def _mode(dtype):
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.manual_seed(1)
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    return RT


def test_batches_reproduce_the_reference_in_parity_mode(cuda):
    """Parity mode, captured graphs: every utterance of the TTS batch (4 texts) and the VC batch (3 waveforms) in every
    case of the fixture -- stops on a probability, at the utterance's own maxlen, and delayed by `threshold` -- has the
    reference's length and its mel / stop probabilities / attention within 1e-3 (the other GPU parity pins' bound), and
    equals its own batch-1 generate_speech(use_cache="graph") within 1e-6."""
    RT = _mode(torch.float32)
    check_against_fixture(synth_model(cuda), synth_fixture(), cuda, 1e-3, "graph")
    RT.dtype = torch.bfloat16


def _tts(cuda, dropout):
    from speecht5_b200.models import T5TransformerModel, make_args
    RT = _mode(torch.bfloat16)
    torch.manual_seed(5)
    tts = T5TransformerModel.build_model(make_args("t5_transformer_base_asr", encoder_layers=2, decoder_layers=2,
                                                   bert_init=True, dprenet_dropout_rate=dropout)).to(cuda).eval()
    with torch.no_grad():
        tts.speech_decoder_postnet.prob_out.bias.fill_(-3.0)
    return RT, tts


def _texts(cuda, lens, seed):
    g = torch.Generator().manual_seed(seed)
    toks = torch.ones(len(lens), max(lens), dtype=torch.long)
    for b, n in enumerate(lens):
        toks[b, :n] = torch.randint(4, 81, (n,), generator=g)
    return toks.to(cuda), torch.tensor(lens), torch.randn(len(lens), 512, generator=g).to(cuda)


def test_bf16_batch_equals_batch_one_and_replays_without_capture(cuda):
    """Throughput mode, prenet dropout off: each utterance of a batch of 5 equals its own batch-1
    generate_speech(use_cache="graph") -- same length, values within 1e-6 relative -- and the rows stop at different
    steps (their own maxlen); a second batch of other texts in the same buckets replays the graphs already captured and
    equals the eager body (lengths, mel, stop probabilities). Probability stops on the graph path: the parity pin."""
    RT, tts = _tts(cuda, 0.0)
    lens = [40, 7, 63, 22, 50]
    toks, src_lengths, spk = _texts(cuda, lens, 1)
    got = tts.generate_speech_batch(src_tokens=toks, src_lengths=src_lengths, spkembs=spk, attention=True)
    for b, n in enumerate(lens):
        alone = tts.generate_speech(src_tokens=toks[b:b + 1, :n], spkembs=spk[b:b + 1], use_cache="graph")
        for g, a in zip(got[b], alone):
            assert g.shape == a.shape, (b, g.shape, a.shape)
            assert rel(g, a) < 1e-6, (b, rel(g, a))
    assert len({m.shape[0] for m, _, _ in got}) == len(lens)
    store = tts._synthesis_graphs
    key = next(k for k in store if k[0] == len(lens))
    n_graphs = len(store[key].graphs)
    toks2, _, spk2 = _texts(cuda, lens, 2)
    again = tts.generate_speech_batch(src_tokens=toks2, src_lengths=src_lengths, spkembs=spk2)
    assert len(store[key].graphs) == n_graphs  # (no new capture)
    eager = tts.generate_speech_batch(src_tokens=toks2, src_lengths=src_lengths, spkembs=spk2,
                                      use_cache="graph_body_eager")
    for x, y in zip(again, eager):
        assert x[0].shape == y[0].shape and x[1].shape == y[1].shape and x[2] is None
        assert rel(x[0], y[0]) < 1e-6 and rel(x[1], y[1]) < 1e-6
    RT.dtype = torch.bfloat16


def test_prenet_dropout_draws_per_row_and_a_seed_reproduces_the_batch(cuda):
    """Always-on prenet dropout: two copies of one text in a batch draw different masks (different frames); the same
    seed gives the same batch again."""
    RT, tts = _tts(cuda, 0.5)
    toks, _, spk = _texts(cuda, [30], 3)
    toks, spk = toks.expand(2, -1).contiguous(), spk.expand(2, -1).contiguous()
    runs = []
    for _ in range(2):
        RT.manual_seed(11)
        runs.append(tts.generate_speech_batch(src_tokens=toks, spkembs=spk, threshold=2.0))
    a, b = runs[0]
    assert a[0].shape == b[0].shape and not torch.equal(a[0], b[0])
    for x, y in zip(runs[0], runs[1]):
        assert torch.equal(x[0], y[0])
    RT.dtype = torch.bfloat16

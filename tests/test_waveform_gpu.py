"""-m gpu: waveform output for ragged batches. st5_lrelu_pad_len against its C contract (exact, NaN sentinels in the
output and in x past every length), HifiGanGenerator.vocode in the release configuration against per-utterance
__call__ (bitwise) and the fp32 oracle, and task.generate_waveform_batch end to end on tiny t2s / s2s models."""
import ctypes as C

import pytest
import torch

from helpers import rel

pytestmark = pytest.mark.gpu

NAN = float("nan")
G = 64  # guard elements around the output


def _lib():
    from speecht5_b200 import _lib
    return _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _want(x, n_in, d, ph, pad, slope, L):
    """The contract in torch: out[b, m] = leaky_relu(x[b, ph + d*m - pad]) for 0 <= src < L[b], else 0 (bf16 of the fp32
    product for negative x)."""
    B, T, Cc = x.shape
    src = ph + d * torch.arange(n_in) - pad
    out = torch.zeros(B, n_in, Cc, dtype=torch.bfloat16)
    for b in range(B):
        ok = (src >= 0) & (src < L[b])
        v = x[b, src[ok]].float()
        out[b, ok] = torch.where(v > 0, v, v * torch.tensor(slope, dtype=torch.float32)).to(torch.bfloat16)
    return out


def _call(x, out, n_in, d, ph, pad, slope, lengths, len_mult, B=None, T=None, Cc=None):
    Bx, Tx, Cx = x.shape if x is not None else out.shape
    return _lib().st5_lrelu_pad_len(_p(x), _p(out), B or Bx, T or Tx, Cc or Cx, n_in, d, ph, pad, slope, _p(lengths),
                                    len_mult, _stream())


@pytest.mark.parametrize("len_mult", [1, 4, 256])
@pytest.mark.parametrize("d", [1, 3, 5])
def test_lrelu_pad_len_contract(cuda, d, len_mult):
    """Every phase of dilation d, k = 7 'same' padding, lengths 0, 1, T, one inside, one past T and a negative one;
    x is NaN at and past each utterance's L_b, the output starts NaN inside NaN guards. lengths = NULL equals
    st5_lrelu_pad bit for bit."""
    B, T, Cc, k = 6, 512, 24, 7
    g = torch.Generator().manual_seed(d * 1000 + len_mult)
    base = (torch.randn(B, T, Cc, generator=g) * 2).to(torch.bfloat16)
    frames = [0, 1, T // len_mult, (T // len_mult) // 2 + 1, T // len_mult + 3, -2]
    L = [max(0, min(f * len_mult, T)) for f in frames]
    assert 0 in L and T in L and len_mult in L
    x = base.clone()
    for b in range(B):
        x[b, L[b]:] = NAN
    xd = x.to(cuda)
    lengths = torch.tensor(frames, dtype=torch.int32, device=cuda)
    pad = (k * d - d) // 2
    for slope in (0.1, 1.0):
        for ph in range(d):
            n_in = (T - ph + d - 1) // d + k - 1
            flat = torch.full((2 * G + B * n_in * Cc,), NAN, dtype=torch.bfloat16, device=cuda)
            out = flat[G:G + B * n_in * Cc].view(B, n_in, Cc)
            assert _call(xd, out, n_in, d, ph, pad, slope, lengths, len_mult) == 0
            torch.cuda.synchronize()
            want = _want(x, n_in, d, ph, pad, slope, L)
            assert torch.equal(out.cpu().view(torch.int16), want.view(torch.int16)), (d, ph, slope)
            assert bool(torch.isnan(torch.cat([flat[:G], flat[-G:]]).float()).all())
            # lengths = NULL: L_b = T, exactly st5_lrelu_pad
            xf = base.to(cuda)
            a = torch.full((B, n_in, Cc), NAN, dtype=torch.bfloat16, device=cuda)
            b_ = torch.full((B, n_in, Cc), NAN, dtype=torch.bfloat16, device=cuda)
            assert _call(xf, a, n_in, d, ph, pad, slope, None, len_mult) == 0
            assert _lib().st5_lrelu_pad(_p(xf), _p(b_), B, T, Cc, n_in, d, ph, pad, slope, _stream()) == 0
            torch.cuda.synchronize()
            assert torch.equal(a.view(torch.int16), b_.view(torch.int16))
            assert torch.equal(a.cpu().view(torch.int16), _want(base, n_in, d, ph, pad, slope, [T] * B).view(torch.int16))


def test_lrelu_pad_len_argument_errors(cuda):
    """-2 for C % 8 != 0, d < 1, ph outside [0, d), len_mult < 1; -3 for a NULL x or out; nothing is written."""
    x = torch.ones(2, 16, 8, dtype=torch.bfloat16, device=cuda)
    x12 = torch.ones(2, 16, 12, dtype=torch.bfloat16, device=cuda)
    out = torch.full((2, 16, 8), NAN, dtype=torch.bfloat16, device=cuda)
    out12 = torch.full((2, 16, 12), NAN, dtype=torch.bfloat16, device=cuda)
    lengths = torch.tensor([3, 16], dtype=torch.int32, device=cuda)
    assert _call(x12, out12, 16, 1, 0, 0, 0.1, lengths, 1) == -2
    for d, ph, mult in ((0, 0, 1), (2, 2, 1), (3, -1, 1), (1, 0, 0), (1, 0, -4)):
        assert _call(x, out, 16, d, ph, 0, 0.1, lengths, mult) == -2, (d, ph, mult)
    assert _call(None, out, 16, 1, 0, 0, 0.1, lengths, 1, B=2, T=16, Cc=8) == -3
    assert _call(x, None, 16, 1, 0, 0, 0.1, lengths, 1) == -3
    torch.cuda.synchronize()
    assert bool(torch.isnan(out.float()).all()) and bool(torch.isnan(out12.float()).all())
    from speecht5_b200 import kernels as K
    with pytest.raises(RuntimeError, match="st5_lrelu_pad_len"):
        K.lrelu_pad_len(x, out, 1, 0, 0, 0.1, lengths, 0)


@pytest.fixture(scope="module")
def release(cuda):
    from oracle.audio_oracle import HifiGanGenerator as Ref
    from speecht5_b200 import vocoder
    torch.manual_seed(0)
    ref = Ref(std=0.02, seed=1).eval()
    with torch.no_grad():
        ref.mean.copy_(torch.randn(80) * 0.5)
        ref.scale.copy_(1.0 + 0.5 * torch.rand(80))
    return ref, vocoder.HifiGanGenerator(ref.state_dict(), device=cuda)


def _mels(lens, seed, cuda):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(L, 80, generator=g) * 1.5 - 2.0).to(cuda) for L in lens]


def test_vocode_ragged_batch_equals_each_utterance(release, cuda):
    """Release configuration: 37, 1, 64, 65 and 200 frames (bucket 256) through one replay equal per-utterance
    __call__ under torch.equal, and are within the 3e-2 relative L2 of the fp32 oracle. A second call in the same
    bucket with other lengths replays the same graph and matches too; NaN in the static input buffer past every length
    changes nothing."""
    ref, gen = release
    lens = [37, 1, 64, 65, 200]
    mels = _mels(lens, 1, cuda)
    got = gen.vocode(mels)
    key = (5, 256, True, str(gen.device))
    assert list(gen._graphs) == [key]
    vg = gen._graphs[key]
    graph = vg.graph
    assert graph is not None and vg.launches > 0
    for b, (m, w) in enumerate(zip(mels, got)):
        alone = gen(m[None])[0]
        assert w.shape == alone.shape == (lens[b] * 256,)
        assert torch.equal(w, alone), (b, (w - alone).abs().max().item())
        with torch.no_grad():
            want = ref(m[None].cpu())[0]
        assert rel(w, want) < 3e-2, (b, rel(w, want))
    lens2 = [200, 129, 3, 64, 150]
    mels2 = _mels(lens2, 2, cuda)
    got2 = gen.vocode(mels2)
    assert list(gen._graphs) == [key] and gen._graphs[key].graph is graph
    for m, w in zip(mels2, got2):
        assert torch.equal(w, gen(m[None])[0])
    # NaN past every length in the static buffer: replay directly (run() would overwrite only the valid frames)
    vg.mel.fill_(NAN)
    for b, m in enumerate(mels):
        vg.mel[b, :m.shape[0]].copy_(m)
    vg.lengths.copy_(torch.tensor(lens, dtype=torch.int32))
    graph.replay()
    torch.cuda.synchronize()
    for b, (L, w) in enumerate(zip(lens, got)):
        assert torch.equal(vg.out[b, :L * 256], w)


def test_vocode_without_normalisation_and_other_batch_sizes(release, cuda):
    """normalize_before=False and B = 1 / 3 get graphs of their own and stay bitwise equal to __call__."""
    _, gen = release
    for lens, norm in (([70], False), ([5, 128, 17], False), ([12, 40, 3], True)):
        mels = _mels(lens, len(lens), cuda)
        for m, w in zip(mels, gen.vocode(mels, normalize_before=norm)):
            assert torch.equal(w, gen(m[None], normalize_before=norm)[0])
    assert (1, 128, False, str(gen.device)) in gen._graphs and (3, 128, False, str(gen.device)) in gen._graphs
    assert (3, 64, True, str(gen.device)) in gen._graphs


@pytest.mark.parametrize("batch", ["tts", "vc"])
def test_generate_waveform_batch_end_to_end(release, cuda, batch):
    """task.generate_waveform_batch on the tiny t2s / s2s model of the batched-synthesis fixture: its mels, stop
    probabilities and attention are exactly generate_speech_batch's (same prenet-dropout seed), its waveforms exactly
    vocode of those mels. threshold=2.0 (the reference's quirk: every length ratio 2.0) gives each utterance a length
    of its own, set by its input length."""
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from test_synth_batch_cpu import batch_inputs, synth_fixture, synth_model
    from types import SimpleNamespace
    _, gen = release
    RT.dtype = torch.bfloat16
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    model = synth_model(cuda)
    task = SpeechT5Task(SimpleNamespace(t5_task="t2s" if batch == "tts" else "s2s"))
    net_input = batch_inputs(synth_fixture(), batch, cuda)
    RT.manual_seed(11)
    want = task.generate_speech_batch([model], net_input, attention=True, threshold=2.0)
    RT.manual_seed(11)
    got = task.generate_waveform_batch([model], net_input, gen, attention=True, threshold=2.0)
    assert len(got) == len(want) == net_input["spkembs"].shape[0]
    assert len({m.shape[0] for m, _, _ in want}) > 1  # ragged
    wavs = gen.vocode([m for m, _, _ in want])
    for (w, mel, probs, attn), (mel0, probs0, attn0), w0 in zip(got, want, wavs):
        assert torch.equal(mel, mel0) and torch.equal(probs, probs0) and torch.equal(attn, attn0)
        assert w.shape == (mel.shape[0] * 256,) and w.dtype == torch.float32
        assert torch.equal(w, w0) and bool(torch.isfinite(w).all())

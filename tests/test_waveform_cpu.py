"""CPU: waveform output for ragged batches (speecht5_b200/vocoder.py HifiGanGenerator.vocode and
task.generate_waveform_batch) -- the length-aware layer code on emulated kernels, the checkpoint names the generator
accepts, and the host-side input checks. The kernels and the captured graph are covered by tests/test_waveform_gpu.py."""
from types import SimpleNamespace

import pytest
import torch

import gemm_emulator

# the reduced configuration of test_frontend_cpu.test_hifigan_device_composition_matches_the_oracle
CFG = dict(model_in_dim=16, upsample_initial_channel=32, upsample_rates=[4, 2], upsample_kernel_sizes=[8, 4],
           resblock_kernel_sizes=[3, 7], resblock_dilation_sizes=[[1, 3], [1, 5]])


def lrelu_pad_len(x, out, d, ph, pad, slope, lengths, len_mult=1):
    """st5_lrelu_pad_len: out[b, m] = leaky_relu(x[b, ph + d*m - pad]) inside [0, L_b), zeros outside, with
    L_b = clamp(lengths[b] * len_mult, 0, T) (lengths None: T)."""
    B, T, C = x.shape
    idx = ph + d * torch.arange(out.shape[1]) - pad
    out.zero_()
    for b in range(B):
        L = T if lengths is None else max(0, min(int(lengths[b]) * len_mult, T))
        ok = (idx >= 0) & (idx < L)
        v = x[b, idx[ok]].float()
        out[b, ok] = torch.where(v > 0, v, v * slope).to(out.dtype)


def _install(monkeypatch):
    from speecht5_b200 import kernels as K
    gemm_emulator.install(monkeypatch)
    monkeypatch.setattr(K, "lrelu_pad_len", lrelu_pad_len)


def _oracle(cfg=CFG):
    from oracle.audio_oracle import HifiGanGenerator as Ref
    torch.manual_seed(0)
    ref = Ref(cfg, std=0.15, seed=1).eval()
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if n.endswith("bias"):
                p.add_(0.05 * torch.randn_like(p))
        ref.mean.copy_(torch.randn(cfg["model_in_dim"]) * 0.1)
        ref.scale.copy_(1.0 + 0.1 * torch.rand(cfg["model_in_dim"]))
    return ref


def test_emulated_kernel_matches_lrelu_pad_without_lengths():
    """The emulation above with lengths = None (or every length >= T) is the existing st5_lrelu_pad emulation."""
    torch.manual_seed(3)
    x = torch.randn(3, 23, 8).to(torch.bfloat16)
    for d, ph, pad, n_in in ((1, 0, 3, 29), (3, 2, 3, 9), (5, 1, 10, 9)):
        want = torch.empty(3, n_in, 8, dtype=torch.bfloat16)
        gemm_emulator.lrelu_pad(x, want, d, ph, pad, 0.1)
        for lengths, mult in ((None, 1), (torch.tensor([23, 30, 99], dtype=torch.int32), 1),
                              (torch.tensor([6, 8, 100], dtype=torch.int32), 4)):
            got = torch.full_like(want, float("nan"))
            lrelu_pad_len(x, got, d, ph, pad, 0.1, lengths, mult)
            assert torch.equal(got, want)


@pytest.mark.parametrize("normalize_before", [True, False])
def test_ragged_batch_equals_each_utterance_alone(monkeypatch, normalize_before):
    """The body vocode captures, run eagerly on emulated kernels: lengths 1, 13, 64 (= the bucket) and 37 in one batch
    padded to 64 frames -- every utterance's waveform equals the emulated __call__ on that utterance alone, although the
    padding frames hold NaN. 13 and 37 are not multiples of the dilations 3 and 5; at the second stage the lengths are
    scaled by 4."""
    from speecht5_b200 import vocoder
    _install(monkeypatch)
    gen = vocoder.HifiGanGenerator(_oracle().state_dict(), CFG, device="cpu")
    lens = [1, 13, 64, 37]
    g = torch.Generator().manual_seed(4)
    mels = [torch.randn(L, 16, generator=g) for L in lens]
    vg = vocoder._VocodeGraph(gen, len(lens), 64, normalize_before, capture=False)
    vg.mel.fill_(float("nan"))
    got = vg.run(mels)
    for b, (m, w) in enumerate(zip(mels, got)):
        alone = gen(m[None], normalize_before)[0]
        assert w.shape == alone.shape == (lens[b] * 8,)
        assert torch.equal(w, alone), (b, (w - alone).abs().max())
    # a second batch of other lengths in the same buffers (the replay of a graph): stale frames are not read either
    lens2 = [64, 2, 5, 50]
    mels2 = [torch.randn(L, 16, generator=g) for L in lens2]
    for m, w in zip(mels2, vg.run(mels2)):
        assert torch.equal(w, gen(m[None], normalize_before)[0])


def test_without_lengths_the_layers_are_unchanged(monkeypatch):
    """_forward(lengths=None) is __call__; lengths equal to T give the same waveform through the length-aware path."""
    from speecht5_b200 import vocoder
    _install(monkeypatch)
    ref = _oracle()
    gen = vocoder.HifiGanGenerator(ref.state_dict(), CFG, device="cpu")
    mel = torch.randn(2, 13, 16)
    base = gen(mel)
    assert torch.equal(gen._forward(mel, True, torch.tensor([13, 13], dtype=torch.int32)), base)
    with torch.no_grad():
        want = ref(mel)
    err = ((base.double() - want.double()).norm() / want.double().norm()).item()
    assert err < 3e-2, err


def _hf_config(tr, cfg=CFG):
    return tr.SpeechT5HifiGanConfig(**cfg)


def test_huggingface_state_dict_and_config(monkeypatch):
    """A random-init transformers.SpeechT5HifiGan: its state dict (`upsampler.{i}` names) and its config dict (with
    keys this generator does not use) build a generator whose output matches the oracle on the same weights -- and the
    oracle on those weights is HuggingFace's own forward."""
    tr = pytest.importorskip("transformers")
    from oracle.audio_oracle import HifiGanGenerator as Ref
    from speecht5_b200 import vocoder
    _install(monkeypatch)
    hf_cfg = _hf_config(tr)
    torch.manual_seed(1)
    hf = tr.SpeechT5HifiGan(hf_cfg).eval()
    with torch.no_grad():
        for n, p in hf.named_parameters():
            p.copy_(torch.randn_like(p) * (0.05 if n.endswith("bias") else 0.15))
        hf.mean.copy_(torch.randn(16) * 0.1)
        hf.scale.copy_(1.0 + 0.1 * torch.rand(16))
    sd = hf.state_dict()
    assert any(k.startswith("upsampler.") for k in sd) and not any(k.startswith("ups.") for k in sd)
    cfg_dict = hf_cfg.to_dict()
    assert "sampling_rate" in cfg_dict and "initializer_range" in cfg_dict
    gen = vocoder.HifiGanGenerator(sd, cfg_dict, device="cpu")
    assert gen.cfg == dict(vocoder.HIFIGAN_CFG, **CFG)
    ref = Ref(CFG).eval()
    ref.load_state_dict({("ups." + k[len("upsampler."):] if k.startswith("upsampler.") else k): v for k, v in sd.items()})
    mel = torch.randn(2, 21, 16)
    with torch.no_grad():
        want = ref(mel)
        assert torch.allclose(hf(mel), want, rtol=1e-5, atol=1e-6)
    got = gen(mel)
    err = ((got.double() - want.double()).norm() / want.double().norm()).item()
    assert err < 3e-2, err
    mels = [mel[0], mel[1, :9]]
    for m, w in zip(mels, vocoder._VocodeGraph(gen, 2, 64, True, capture=False).run(mels)):
        assert torch.equal(w, gen(m[None])[0])


def test_weight_norm_pairs_fold_like_torch_weight_norm(monkeypatch):
    """A reference-shaped state dict with weight_g / weight_v pairs (`ups.{i}`, no mean / scale) folds to the weights
    oracle.audio_oracle.fold_weight_norm gives, and torch.nn.utils.weight_norm's own weight; HuggingFace names fold the
    same way, and the generator builds from it (mean 0, scale 1)."""
    from oracle.audio_oracle import fold_weight_norm
    from speecht5_b200 import vocoder
    g = torch.Generator().manual_seed(7)
    sd = {}
    for k, v in _oracle().state_dict().items():
        if k.endswith(".weight"):
            base = k[:-len("weight")]
            sd[base + "weight_g"] = torch.rand((v.shape[0],) + (1,) * (v.dim() - 1), generator=g) + 0.5
            sd[base + "weight_v"] = torch.randn(v.shape, generator=g)
        elif k not in ("mean", "scale"):
            sd[k] = v
    want = fold_weight_norm(sd)
    got = vocoder.plain_state_dict(sd)
    assert set(got) == set(want)
    for k in want:
        assert torch.allclose(got[k], want[k], rtol=2e-6, atol=0), k
    # torch.nn.utils.weight_norm's own weight for one conv
    conv = torch.nn.ConvTranspose1d(32, 16, 8, 4, padding=2)
    wn = torch.nn.utils.weight_norm(conv)
    with torch.no_grad():
        wn.weight_g.copy_(sd["ups.0.weight_g"])
        wn.weight_v.copy_(sd["ups.0.weight_v"])
        wn(torch.zeros(1, 32, 3))  # (the hook recomputes .weight)
    assert torch.allclose(got["ups.0.weight"], wn.weight, rtol=2e-6, atol=0)
    other = vocoder.plain_state_dict({("upsampler." + k[4:] if k.startswith("ups.") else k): v for k, v in sd.items()})
    assert set(other) == set(got) and all(torch.equal(other[k], got[k]) for k in got)
    _install(monkeypatch)
    gen = vocoder.HifiGanGenerator(sd, CFG, device="cpu")
    assert torch.equal(gen.mean, torch.zeros(16)) and torch.equal(gen.scale, torch.ones(16))
    assert gen(torch.randn(1, 5, 16)).shape == (1, 40)


def _no_launch(monkeypatch):
    from speecht5_b200 import kernels as K

    def boom(*a, **k):
        raise AssertionError("a kernel was launched")
    for name in ("gemm", "lrelu_pad", "lrelu_pad_len", "cast_bf16"):
        monkeypatch.setattr(K, name, boom)


def test_host_validation_raises_before_any_launch(monkeypatch):
    from speecht5_b200 import vocoder
    from speecht5_b200.tasks import SpeechT5Task
    _install(monkeypatch)
    gen = vocoder.HifiGanGenerator(_oracle().state_dict(), CFG, device="cpu")
    _no_launch(monkeypatch)
    ok = torch.randn(5, 16)
    bad = [[], (), ok, [ok, torch.randn(5, 15)], [torch.randn(5)], [torch.randn(0, 16)], [ok, ok.double()],
           [ok.bfloat16()], [ok, torch.empty(5, 16, device="meta")], [ok, "mel"]]
    for mels in bad:
        with pytest.raises(ValueError):
            gen.vocode(mels)
    # the task call checks the batch, the device and the mel width before synthesis
    task = SpeechT5Task(SimpleNamespace(t5_task="t2s"))

    class Model:
        speech_decoder_postnet = SimpleNamespace(odim=16)

        def generate_speech_batch(self, **kw):
            raise AssertionError("synthesis ran")
    toks = torch.randint(4, 81, (2, 7))
    for net_input, model in (({"src_tokens": toks[:0]}, Model()), ({"src_tokens": toks[:, :0]}, Model()),
                             ({"src_tokens": toks.to("meta")}, Model()), ({}, Model())):
        with pytest.raises(ValueError):
            task.generate_waveform_batch([model], net_input, gen)
    wide = Model()
    wide.speech_decoder_postnet = SimpleNamespace(odim=80)
    with pytest.raises(ValueError):
        task.generate_waveform_batch([wide], {"src_tokens": toks}, gen)

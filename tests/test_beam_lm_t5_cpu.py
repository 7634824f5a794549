"""LM shallow fusion with SpeechT5's own LM architecture (`transformer_lm_t5`: heads of 80 channels, rows up to 2048
wide) without a GPU: the reference SequenceGenerator's hypotheses with a tiny transformer_lm_t5 fused in
(tests/golden/ref_beam_lm_t5_tiny.npz, make_golden_beam_lm_t5.py) reproduced by the host composition on emulated
kernels, with the head-dimension-general entry points (st5_attn_decode_hd_fwd / st5_attn_lineage_hd_fwd) stood in for
below; the LM's forward at head dim 80 against the reference LM's log-probabilities; the preset against the reference's
arch function; what stays rejected; and the new kernels' register budget."""
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
import gemm_emulator
from test_beam_cpu import MASK_KW, V, check_hypos, model, src  # noqa: F401  (model: the fixture of the ASR model)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
N_CASES = 5

from speecht5_b200 import ops as _ops  # noqa: E402

_REAL_ATTENTION = _ops.attention  # (captured before any test patches it)


# ------------------------------------------------------------------------------------ head-dim-general CPU stand-ins
def attn_decode_hd_fwd(q, k, v, out, *, H, head_dim, scale, key_pad=None, probs=None):
    """st5_attn_decode_hd_fwd in fp64: one query row per batch row over its own keys; a row whose keys are all masked
    gives zeros, as the kernels do."""
    assert head_dim in (64, 80)
    B, Tk = k.shape[0], k.shape[1]
    qh = q[:, 0].double().reshape(B, H, head_dim)
    s = torch.einsum("bhc,bjhc->bhj", qh, k.double().reshape(B, Tk, H, head_dim)) * scale
    if key_pad is not None:
        s = s.masked_fill(key_pad.bool()[:, None], float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    out.copy_(torch.einsum("bhj,bjhc->bhc", p, v.double().reshape(B, Tk, H, head_dim)).reshape(out.shape).to(out.dtype))
    if probs is not None:
        probs.copy_(p.reshape(probs.shape).float())


def attn_lineage_hd_fwd(q, k, v, out, *, H, head_dim, scale, key_pad=None, kv_rows=None, kv_div=1):
    """st5_attn_lineage_hd_fwd: key / value j of query row b gathered from row kv_rows[b, j] or b // kv_div."""
    B, Tk = q.shape[0], k.shape[1]
    if kv_rows is not None:
        rows = kv_rows[:, :Tk].long()
        j = torch.arange(Tk)[None].expand(B, Tk)
        kg, vg = k[rows, j], v[rows, j]
    else:
        idx = torch.arange(B) // kv_div
        kg, vg = k[idx], v[idx]
    attn_decode_hd_fwd(q, kg, vg, out, H=H, head_dim=head_dim, scale=scale, key_pad=key_pad)


def ln_fwd_wide(x, residual, gamma, beta, y, mean=None, rstd=None, eps=1e-5):
    """st5_ln_fwd_wide: y = LayerNorm(x + residual) in fp64."""
    s = x.double() + (residual.double() if residual is not None else 0.0)
    y.copy_(torch.nn.functional.layer_norm(s, (s.shape[-1],), gamma.double(), beta.double(), eps).to(y.dtype))


def install(monkeypatch):
    """The stand-ins above; ops.attention stays the package's own for heads that are not 64 wide (so its route through
    ops.attention_rows is what runs), and is tests/gemm_emulator.py's torch statement for the speech model's heads."""
    from speecht5_b200 import kernels as K, ops
    monkeypatch.setattr(K, "attn_decode_hd_fwd", attn_decode_hd_fwd)
    monkeypatch.setattr(K, "attn_lineage_hd_fwd", attn_lineage_hd_fwd)
    monkeypatch.setattr(K, "ln_fwd_wide", ln_fwd_wide)

    def attention(q_buf, kv_buf, *, H, d, **kw):
        if d != 64 * H:
            return _REAL_ATTENTION(q_buf, kv_buf, H=H, d=d, **kw)
        return gemm_emulator.attention(q_buf, kv_buf, H=H, d=d, **kw)
    monkeypatch.setattr(ops, "attention", attention)


# ------------------------------------------------------------------------------------------------------- fixture
@pytest.fixture(autouse=True)
def _keep_global_rng():
    """Leave torch's global generator as each test found it (the tests below seed it), so that the tests after these
    draw what they would without them."""
    state = torch.get_rng_state()
    yield
    torch.set_rng_state(state)


def load():
    return dict(np.load(os.path.join(GOLD, "ref_beam_lm_t5_tiny.npz")))


def lm_args(blob, arch=True):
    L, C, H, F, tps = (int(x) for x in blob["lm_args"])
    a = Namespace(decoder_layers=L, decoder_embed_dim=C, decoder_attention_heads=H, decoder_ffn_embed_dim=F,
                  tokens_per_sample=tps)
    if arch:
        a.arch = "transformer_lm_t5"
    return a


def lm_state(blob):
    return {k[3:]: torch.from_numpy(v).float() for k, v in blob.items() if k.startswith("lm/")}


def build_lm(blob):
    from speecht5_b200.lm import TransformerLM
    lm = TransformerLM(lm_args(blob), V - 2)
    lm.load_fairseq_state(lm_state(blob))
    return lm


def fake_fairseq_lm(blob):
    inner = build_lm(blob)
    m = torch.nn.Module()
    m.decoder = inner.decoder
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
    install(monkeypatch)
    m, _ = model
    yield m, build_lm(load()), load()


def _reference_or_skip():
    from oracle import ref_loader as rl
    if not rl.available():
        pytest.skip("reference tree not available")
    sys.path.insert(0, GOLD)
    import make_golden_beam_lm_t5 as mg
    return mg


# ------------------------------------------------------------------------------------------------------- tests
def test_fixture_is_what_the_reference_produces_now():
    mg = _reference_or_skip()
    fresh, blob = mg.make(), load()
    assert sorted(fresh) == sorted(blob)
    for k in blob:
        assert np.array_equal(fresh[k], blob[k]), k


@pytest.mark.parametrize("given", [
    {}, dict(decoder_embed_dim=160, decoder_attention_heads=2, decoder_layers=2, decoder_ffn_embed_dim=256),
    dict(activation_fn="relu", dropout=None, share_decoder_input_output_embed=True),
    dict(no_tie_adaptive_proj=False), dict(decoder_final_norm=False), dict(decoder_output_dim=640)])
def test_preset_equals_the_reference_arch_function(given):
    from speecht5_b200.lm import transformer_lm_t5
    mg = _reference_or_skip()
    want = Namespace(**given)
    mg.arch_fn()(want)
    got = transformer_lm_t5(Namespace(**given))
    assert vars(got) == vars(want)


def test_preset_sizes_and_the_arch_switch():
    from speecht5_b200.lm import TransformerLM, transformer_lm_t5
    a = transformer_lm_t5(Namespace())
    assert (a.decoder_layers, a.decoder_embed_dim, a.decoder_attention_heads, a.decoder_ffn_embed_dim,
            a.activation_fn, a.decoder_normalize_before) == (20, 1280, 16, 6144, "gelu", True)
    blob = load()
    lm = TransformerLM(lm_args(blob), V - 2)
    assert lm.args.activation_fn == "gelu" and lm.decoder.layers[0].self_attn.head_dim == 80
    # without the arch name the same sizes take base_lm_architecture's relu
    assert TransformerLM(lm_args(blob, arch=False), V - 2).args.activation_fn == "relu"


def test_lm_matches_the_reference_log_probabilities(fused):
    """TransformerLM.forward at head dim 80: ops.attention_rows (B*T one-row queries, kv_div = T, causal key mask)."""
    _, lm, blob = fused
    tok = torch.from_numpy(blob["probe/tokens"])
    got = lm.log_probs(tok)
    want = torch.from_numpy(blob["probe/lprobs"])
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=0, atol=2e-4), float((got - want).abs().max())


def test_load_lm_and_from_fairseq_with_the_arch(fused, tmp_path):
    from speecht5_b200.lm import TransformerLM, load_lm
    _, lm, blob = fused
    want = lm.state_dict()

    def same(other):
        got = other.state_dict()
        assert sorted(got) == sorted(want)
        for k in want:
            assert torch.equal(got[k], want[k]), k
        assert other.args.activation_fn == "gelu"
    fs = fake_fairseq_lm(blob)
    same(TransformerLM.from_fairseq(fs))
    state = dict(fs.state_dict(), **{"decoder.embed_positions._float_tensor": torch.zeros(1)})
    torch.save({"model": state, "args": lm_args(blob)}, tmp_path / "args.pt")
    torch.save({"model": state, "cfg": {"model": vars(lm_args(blob))}}, tmp_path / "cfg.pt")
    same(load_lm(str(tmp_path / "args.pt")))
    same(load_lm(str(tmp_path / "cfg.pt")))


def test_generate_text_beam_with_the_t5_lm_matches_the_reference(fused):
    m, lm, blob = fused
    source, pm = src(dict(np.load(os.path.join(GOLD, "ref_beam_tiny.npz"))))
    for ci, K, mn, mx, lp, w in cases(blob):
        got = m.generate_text_beam(source, pm, beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, use_cache=True,
                                   lm=lm, lm_weight=w, **MASK_KW)
        check_hypos(got, blob, ci)
    ci, K, mn, mx, lp, w = list(cases(blob))[2]
    for b in range(source.shape[0]):
        one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp,
                                   lm=lm, lm_weight=w, **MASK_KW)
        check_hypos(one, blob, ci, rows=[b])


def test_generators_with_the_t5_lm(fused):
    from speecht5_b200.generator import BeamSearchGenerator
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
    args = SimpleNamespace(beam=K, max_len_a=0, max_len_b=mx, min_len=1, unnormalized=False, lenpen=1.0, unkpen=0.0)
    g = task.build_generator([m], args, seq_gen_cls=BeamSearchGenerator,
                             extra_gen_cls_kwargs={"lm_model": fs, "lm_weight": w})
    check_hypos(task.inference_step(g, [m], sample), blob, 2)


def test_attention_decode_routes_by_head_width(monkeypatch):
    """ops.attention_decode: 64-wide heads on the original entry points (unchanged calls), 80-wide on the _hd ones."""
    from speecht5_b200 import kernels as K, ops
    calls = []
    for name in ("attn_decode_fwd", "attn_lineage_fwd", "attn_decode_hd_fwd", "attn_lineage_hd_fwd"):
        monkeypatch.setattr(K, name, lambda *a, _n=name, **kw: calls.append((_n, kw.get("head_dim"))))
    for hd in (64, 80):
        q = torch.zeros(2, 1, 3 * 2 * hd)
        ops.attention_decode(q, None, H=2, d=2 * hd, q_col=0, k_col=1, v_col=2, scale=1.0)
        ops.attention_decode(q, None, H=2, d=2 * hd, q_col=0, k_col=1, v_col=2, scale=1.0, kv_div=2)
    assert calls == [("attn_decode_fwd", None), ("attn_lineage_fwd", None), ("attn_decode_hd_fwd", 80),
                     ("attn_lineage_hd_fwd", 80)]
    with pytest.raises(AssertionError):
        ops.attention_decode(torch.zeros(2, 1, 96), None, H=1, d=32, q_col=0, k_col=1, v_col=2, scale=1.0)


def test_wide_layer_norm_route(monkeypatch):
    """C > 1024: st5_ln_fwd_wide without a gradient, NotImplementedError with one."""
    from speecht5_b200 import kernels as K, ops
    monkeypatch.setattr(K, "ln_fwd_wide", ln_fwd_wide)
    torch.manual_seed(0)
    ln = torch.nn.LayerNorm(1280)
    torch.nn.init.normal_(ln.weight)
    torch.nn.init.normal_(ln.bias)
    x, r = torch.randn(3, 5, 1280), torch.randn(3, 5, 1280)
    with torch.no_grad():
        y = ops.residual_layer_norm(x, r, ln)
        assert torch.allclose(y, ln(x + r), atol=1e-5)
    with pytest.raises(NotImplementedError):
        ops.residual_layer_norm(x, None, ln)  # (ln's parameters require a gradient)


@pytest.mark.parametrize("C,H", [(64, 2), (160, 5), (2560, 32), (1280, 40)])
def test_other_head_widths_and_rows_past_2048_raise(C, H):
    from speecht5_b200.lm import TransformerLM
    args = Namespace(decoder_layers=1, decoder_embed_dim=C, decoder_attention_heads=H, decoder_ffn_embed_dim=128)
    with pytest.raises(NotImplementedError):
        TransformerLM(args, 10)


def test_the_speech_model_keeps_64_wide_heads():
    from speecht5_b200.models.modules.transformer import MultiheadAttention
    with pytest.raises(AssertionError):
        MultiheadAttention(160, 2)
    assert MultiheadAttention(160, 2, head_dims=(64, 80)).head_dim == 80


def test_new_kernels_fit_their_launch_bounds_without_spills():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("cuobjdump or library not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    seen = set()
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res):
        name, regs, stack, local = m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))
        if "80_split" in name or "80_combine" in name or "ln_fwd_wide" in name:
            assert stack == 0 and local == 0 and regs * 128 <= 65536, (name, regs, stack, local)
            seen.add(name)
    assert len(seen) == 7, sorted(seen)  # (decode / lineage x fp32 / bf16, the combine, LayerNorm x 2 dtypes)

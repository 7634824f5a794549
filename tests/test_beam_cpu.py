"""Beam search for text output (T5TransformerModel.generate_text_beam, generator.BeamSearchGenerator) without a GPU:
the reference SequenceGenerator's own hypotheses (tests/golden/ref_beam_tiny.npz, make_golden_beam.py) reproduced by the
torch statement tests/beam_ref.py and by the host composition (incremental.BeamGraph) on emulated kernels; the C ABI of
the three new entry points (struct layout, argument errors) and their register budget."""
import ctypes as C
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import beam_emulator
import beam_ref
import gemm_emulator

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
V = 81


def load():
    return dict(np.load(os.path.join(GOLD, "ref_beam_tiny.npz")))


def cases(blob):
    for ci in range(4):
        K, mn, mx = (int(x) for x in blob[f"c{ci}/meta"])
        yield ci, K, mn, mx, float(blob[f"c{ci}/len_penalty"])


@pytest.fixture
def model(monkeypatch):
    from helpers import NO_DROPOUT, TINY
    from speecht5_b200 import frontend
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    gemm_emulator.install(monkeypatch)
    beam_emulator.install(monkeypatch)
    monkeypatch.setattr(RT, "dtype", torch.float32)
    from test_frontend_cpu import _cpu_extractor_forward
    monkeypatch.setattr(frontend.ConvFeatureExtractor, "forward", _cpu_extractor_forward)
    RT.invalidate_shadows()
    blob = load()
    over = dict(TINY, **NO_DROPOUT, bert_init=True, build_speech_encoder=True, build_text_decoder=True,
                conv_feature_layers="[(32, 10, 5)] + [(32, 3, 2)] * 4 + [(32, 2, 2)] * 2", feature_grad_mult=1.0,
                conv_pos=16, conv_pos_groups=4, use_conv_pos=True, use_sinc_pos=True, mask_prob=0.0,
                mask_channel_prob=0.0, max_text_positions=600)
    m = T5TransformerModel.build_model(make_args("t5_transformer_base_asr", **over)).eval()
    m.load_state_dict({k[6:]: torch.from_numpy(v) for k, v in blob.items() if k.startswith("state/")}, strict=False)
    yield m, blob
    RT.invalidate_shadows()


def check_hypos(got, blob, ci, rows=None, tol=1e-4):
    rows = range(len(got)) if rows is None else rows
    for b, hs in zip(rows, got):
        K = blob[f"c{ci}/len"].shape[1]
        assert len(hs) == K, (ci, b)
        for i, h in enumerate(hs):
            n = int(blob[f"c{ci}/len"][b, i])
            assert h["tokens"].tolist() == blob[f"c{ci}/tokens"][b, i, :n].tolist(), (ci, b, i)
            assert abs(float(h["score"]) - float(blob[f"c{ci}/score"][b, i])) <= tol, (ci, b, i)
            want = torch.from_numpy(blob[f"c{ci}/pos"][b, i, :n])
            # (differences of cumulative fp32 scores: the error scales with the largest cumulative magnitude)
            atol = tol * (1.0 + float(want.cumsum(0).abs().max()))
            assert torch.allclose(h["positional_scores"].float().cpu(), want, rtol=tol, atol=atol), (ci, b, i)
            assert h["attention"] is None


def src(blob):
    return torch.from_numpy(blob["in/source"]), torch.from_numpy(blob["in/padding_mask"])


MASK_KW = dict(blank=V - 1, mask_idx=V - 2)


def test_fixture_is_what_the_reference_produces_now():
    from oracle import ref_loader as rl
    if not rl.available():
        pytest.skip("reference tree not available")
    sys.path.insert(0, GOLD)
    import make_golden_beam as mg
    fresh, blob = mg.make(), load()
    assert sorted(fresh) == sorted(blob)
    for k in blob:
        assert np.array_equal(fresh[k], blob[k]), k


def test_beam_ref_search_reproduces_the_fixture(model):
    m, blob = model
    source, pm = src(blob)
    enc = m.forward_encoder(source, padding_mask=pm)
    mask = torch.zeros(V)
    mask[1], mask[V - 1], mask[V - 2] = -float("inf"), -float("inf"), -float("inf")
    for ci, K, mn, mx, lp in cases(blob):
        B = source.shape[0]
        idx = torch.arange(B).repeat_interleave(K)
        encK = dict(enc, encoder_out=[enc["encoder_out"][0][:, idx]],
                    encoder_padding_mask=[enc["encoder_padding_mask"][0][idx]])
        encK.pop("_encoder_out_btc", None)

        def logits_fn(tokens):
            with torch.no_grad():
                out, _ = m.forward_decoder(tokens, encK, incremental_state={})
            return out[:, -1, :].float()
        got = beam_ref.search(logits_fn, B, K, V, mx, min_len=mn, mask=mask, len_penalty=lp)
        check_hypos(got, blob, ci)


def test_generate_text_beam_on_emulated_kernels_matches_the_reference(model):
    m, blob = model
    source, pm = src(blob)
    for ci, K, mn, mx, lp in cases(blob):
        got = m.generate_text_beam(source, pm, beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp, use_cache=True,
                                   **MASK_KW)
        check_hypos(got, blob, ci)
    # each sentence alone (batch 1) gives its own hypotheses
    ci, K, mn, mx, lp = next(iter(cases(blob)))
    for b in range(source.shape[0]):
        one = m.generate_text_beam(source[b:b + 1], pm[b:b + 1], beam_size=K, max_len_b=mx, min_len=mn, len_penalty=lp,
                                   **MASK_KW)
        check_hypos(one, blob, ci, rows=[b])
    with pytest.raises(ValueError, match="True or 'graph'"):
        m.generate_text_beam(source, pm, use_cache=False)


def test_beam_search_generator_and_build_generator(model):
    from types import SimpleNamespace
    from speecht5_b200.generator import BeamSearchGenerator, GreedyGenerator
    from speecht5_b200.tasks.speecht5 import SpeechT5Task
    m, blob = model
    source, pm = src(blob)
    sample = {"net_input": {"source": source, "padding_mask": pm}}
    vocab = SimpleNamespace(pad=lambda: 1, eos=lambda: 2, unk=lambda: 3)
    g1 = BeamSearchGenerator([m], vocab, beam_size=1, max_len_b=16, use_cache=True, **MASK_KW).generate([m], sample)
    gg = GreedyGenerator([m], vocab, max_len_b=16, use_cache=True, **MASK_KW).generate([m], sample)
    for a, b in zip(g1, gg):
        assert len(a) == 1 and a[0]["tokens"].tolist() == b[0]["tokens"].tolist()
        assert torch.equal(a[0]["positional_scores"], b[0]["positional_scores"])
    with pytest.raises(NotImplementedError):
        BeamSearchGenerator([m], vocab, beam_size=5, ctc_weight=0.3)
    task = SpeechT5Task.__new__(SpeechT5Task)
    task.args, task.dicts = SimpleNamespace(ctc_weight=0.0), {"text": vocab}
    task.blank_symbol_idx, task.mask_idx = V - 1, V - 2
    args = SimpleNamespace(beam=5, max_len_a=0, max_len_b=16, min_len=1, unnormalized=False, lenpen=1.0, unkpen=0.0)
    gen = task.build_generator([m], args, seq_gen_cls=BeamSearchGenerator)
    hypos = task.inference_step(gen, [m], sample)
    check_hypos(hypos, blob, 1)
    with pytest.raises(NotImplementedError):
        task.inference_step(gen, [m], sample, prefix_tokens=torch.zeros(4, 1, dtype=torch.long))


def test_lineage_struct_layout_matches_the_header(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    from speecht5_b200 import _lib
    prog = tmp_path / "lay.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "speecht5_b200.h"\nint main(void){printf("%zu %zu '
                    '%zu %zu\\n", sizeof(st5_attn_lineage_args), offsetof(st5_attn_lineage_args, kv_rows), '
                    'offsetof(st5_attn_lineage_args, kv_rows_ld), offsetof(st5_attn_lineage_args, kv_div));return 0;}\n')
    exe = tmp_path / "lay"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    A = _lib.AttnLineageArgs
    assert got == [C.sizeof(A), A.kv_rows.offset, A.kv_rows_ld.offset, A.kv_div.offset]


def test_argument_errors_are_reported_without_a_device():
    from speecht5_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    lib = _lib.load()
    one = C.c_void_p(16)
    topk = lambda K, V, ld, p=one: lib.st5_beam_topk(p, ld, 0, 1, K, V, p, p, 1.0, 2, p, p, p, p, p, p, p, None)  # noqa
    assert topk(17, 81, 81) == -2 and b"st5_beam_topk" in lib.st5_last_error()
    assert topk(2, 0, 81) == -2 and topk(2, 40000, 40000) == -2
    assert topk(2, 81, 81, p=None) == -3 and topk(2, 81, 80) == -6
    upd = lambda K, T, p=one: lib.st5_beam_update(1, K, 81, T, 2, p, p, 1, 1.0, *([p] * 17), None)  # noqa
    assert upd(17, 64) == -2 and upd(2, 1) == -2 and upd(2, 64, p=None) == -3
    assert lib.st5_beam_update(1, 4, 4, 64, 2, one, one, 1, 1.0, *([one] * 17), None) == -2  # (V <= K)
    a = _lib.AttnLineageArgs()
    a.base.B, a.base.H, a.base.Tk, a.base.k, a.base.v, a.kv_div = 1, 1, 8, 16, 16, 0
    assert lib.st5_attn_lineage_fwd(C.byref(a), None) == -2
    a.kv_div, a.base.k = 1, 8
    assert lib.st5_attn_lineage_fwd(C.byref(a), None) == -6


def test_beam_kernels_fit_their_launch_bounds_without_spills():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None or not os.path.exists(LIB):
        pytest.skip("cuobjdump or library not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    seen = set()
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res):
        name, regs, stack, local = m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))
        if re.search(r"beam_|attn_lineage_", name):
            assert stack == 0 and local == 0 and regs * 256 <= 65536, (name, regs, stack, local)
            seen.add(name)
    assert len(seen) == 7, sorted(seen)

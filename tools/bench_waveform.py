"""Waveform output for batched speech synthesis (task.generate_waveform_batch) on one GPU: Base model in bf16 with
random weights, the release HiFi-GAN configuration with random weights, CUDA-event timed after a warm-up call that
captures the graphs. Steps are fixed by threshold=2.0 (as in tools/bench_synth_batch.py: every utterance runs exactly
T_enc decoder steps), so the mel lengths do not depend on an untrained model's stop flag.
  * TTS: 160-token texts with x-vectors at B = 1, 8, 32;
  * VC: 8 sources of 3 s.
Per workload: synthesis ms (generate_speech_batch), vocode ms (one graph replay) against the per-utterance eager
__call__ loop on the same mels, library launches per call (kernels.LAUNCHES; for vocode, the launches the captured
pass holds), waveform samples / s and real-time factor (audio seconds at 16 kHz per wall second) of synthesis + vocode,
and the peak memory above the resident model and vocoder. Prints one JSON line with the card's name and power limit.
usage: python tools/bench_waveform.py [--reps 3]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_vc import card  # noqa: E402

SAMPLE_RATE = 16000


def _time(fn, reps):
    import torch
    r = fn()  # capture / warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from oracle.audio_oracle import HifiGanGenerator as Ref
    from speecht5_b200 import kernels as K
    from speecht5_b200 import vocoder
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    assert torch.cuda.is_available(), "bench_waveform measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    margs = make_args("t5_transformer_base_asr", bert_init=True, build_speech_encoder=True, t5_task="s2s",
                      max_speech_positions=1876)
    task = SpeechT5Task(margs)
    model = task.build_model(margs).to(dev).eval()
    gen = vocoder.HifiGanGenerator(Ref(std=0.01, seed=7).eval().state_dict(), device=dev)
    hop = gen.hop
    g = torch.Generator().manual_seed(1)
    out = {"metric": "waveform_batch", "dtype": "bf16", "threshold": 2.0, "sample_rate": SAMPLE_RATE}

    def row(name, net_input):
        B = net_input["spkembs"].shape[0]
        synth_ms, res = _time(lambda: task.generate_speech_batch([model], net_input, threshold=2.0), args.reps)
        mels = [m for m, _, _ in res]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        voc_ms, wavs = _time(lambda: gen.vocode(mels), args.reps)
        peak = torch.cuda.max_memory_allocated(dev) - base
        vg = next(v for k, v in gen._graphs.items() if k[0] == B and k[1] >= max(m.shape[0] for m in mels))
        loop_ms, _ = _time(lambda: [gen(m[None]) for m in mels], args.reps)
        n0 = K.LAUNCHES
        [gen(m[None]) for m in mels]
        loop_launches = K.LAUNCHES - n0
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        e2e_ms, got = _time(lambda: task.generate_waveform_batch([model], net_input, gen, threshold=2.0), args.reps)
        e2e_peak = torch.cuda.max_memory_allocated(dev) - base
        samples = sum(w.numel() for w in wavs)
        assert samples == sum(w.numel() for w, _, _, _ in got)
        out[name] = {"B": B, "mel_frames": [min(m.shape[0] for m in mels), max(m.shape[0] for m in mels)],
                     "T_bucket": vg.T, "synthesis_ms": round(synth_ms, 2), "vocode_ms": round(voc_ms, 2),
                     "eager_loop_ms": round(loop_ms, 2), "vocode_speedup": round(loop_ms / voc_ms, 2),
                     "vocode_launches_per_call": vg.launches, "eager_loop_launches": loop_launches,
                     "end_to_end_ms": round(e2e_ms, 2), "samples_per_s": round(samples * 1000.0 / e2e_ms),
                     "rtf": round(e2e_ms / 1000.0 / (samples / SAMPLE_RATE), 4),
                     "vocode_samples_per_s": round(samples * 1000.0 / voc_ms),
                     "vocode_peak_mib": round(peak / 2 ** 20, 1), "end_to_end_peak_mib": round(e2e_peak / 2 ** 20, 1)}

    for B in (1, 8, 32):
        toks = torch.randint(4, 81, (B, 160), generator=g).to(dev)
        spk = torch.randn(B, 512, generator=g).to(dev)
        row(f"tts_160tok_B{B}", {"src_tokens": toks, "spkembs": spk})
    src = (torch.randn(8, 48_000, generator=g) * 0.1).to(dev)
    row("vc_3s_B8", {"source": src, "padding_mask": torch.zeros_like(src, dtype=torch.bool),
                     "spkembs": torch.randn(8, 512, generator=g).to(dev)})
    out["resident_mib"] = round(torch.cuda.memory_allocated(dev) / 2 ** 20, 1)
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

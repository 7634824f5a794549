"""Measurement of the inference-side rows (SURVEY 8a rows 15, 16, 21) on one GPU, CUDA-event timed after a
warm-up: greedy synthesis with prefix recomputation vs the key/value cache (fixed number of decoder steps), the HiFi-GAN
generator and the log-mel front end, each with the CPU oracle timed next to it on a small sample.
usage: python tools/bench_inference.py [--steps 100] > bench_inference.json"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def cuda_ms(fn, reps=3):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100, help="decoder steps of the synthesis runs (2 mel frames each)")
    args = ap.parse_args()
    import torch
    from speecht5_b200 import audio, vocoder
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    dev = torch.device("cuda", 0)
    RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    out = {}
    # ---- row 21 (TTS half): synthesis of a fixed number of steps (threshold 2.0 can never fire -> runs to maxlen; the
    # reference's knob reuse makes maxlen = int(T_text * threshold / r), so pick the text length accordingly)
    margs = make_args("t5_transformer_base_asr", encoder_layerdrop=0.0, decoder_layerdrop=0.0, bert_init=True)
    model = T5TransformerModel.build_model(margs).to(dev).eval()
    T_text = args.steps  # maxlen = int(T_text * 2.0 / 2) = T_text
    tok = torch.randint(4, 81, (1, T_text), device=dev)
    spk = torch.randn(1, 512, device=dev)
    for name, kw in (("prefix", {}), ("kv_cache", dict(use_cache=True)), ("kv_cache_graph", dict(use_cache="graph"))):
        ms = cuda_ms(lambda: model.generate_speech(src_tokens=tok, spkembs=spk, threshold=2.0, **kw), reps=2)
        out[f"generate_speech_{name}"] = dict(ms=ms, decoder_steps=args.steps, ms_per_step=ms / args.steps)
    # ---- row 21 (ASR half): beam-1 text decoding of 8 x 10 s waveforms, a fixed number of steps (eos forbidden until
    # min_len = the step budget), encoder included: prefix recomputation / eager key-value cache / one graph per step
    del model
    aargs = make_args("t5_transformer_base_asr", build_speech_encoder=True, build_text_decoder=True, bert_init=True,
                      encoder_layerdrop=0.0, decoder_layerdrop=0.0, max_text_positions=600)
    asr = T5TransformerModel.build_model(aargs).to(dev).eval()
    wav = torch.randn(8, 160000, device=dev) * 0.1
    wpm = torch.zeros(8, 160000, dtype=torch.bool, device=dev)
    nsteps = min(args.steps, 100)
    for name, uc in (("prefix", False), ("kv_cache", True), ("kv_cache_graph", "graph")):
        ms = cuda_ms(lambda: asr.generate_text_greedy(wav, wpm, max_len_b=nsteps, min_len=nsteps, use_cache=uc), reps=2)
        out[f"greedy_text_{name}"] = dict(ms=ms, utterances=8, decoder_steps=nsteps + 1, ms_per_step=ms / (nsteps + 1),
                                          utt_per_s=8 / (ms / 1e3))
    del asr
    # ---- row 16: HiFi-GAN, 8 s of audio per utterance (500 frames), batch 4
    from oracle.audio_oracle import HifiGanGenerator as Ref, logmelfilterbank as ref_logmel
    ref = Ref(std=0.02, seed=1).eval()
    gen = vocoder.HifiGanGenerator(ref.state_dict(), device=dev)
    mel = torch.randn(4, 500, 80, device=dev)
    ms = cuda_ms(lambda: gen(mel))
    sec_audio = 4 * 500 * 256 / 16000.0
    out["hifigan"] = dict(ms=ms, audio_seconds=sec_audio, realtime_factor=sec_audio / (ms / 1e3),
                          tflops=4 * 218.65e9 * (500 / 800.0) / (ms / 1e3) / 1e12)
    t0 = time.time()
    with torch.no_grad():
        ref(torch.randn(1, 50, 80))
    out["hifigan"]["cpu_oracle_realtime_factor"] = (50 * 256 / 16000.0) / (time.time() - t0)
    # ---- row 15: log-mel of 32 x 10 s
    wav = torch.randn(32, 160000, device=dev) * 0.1
    ms = cuda_ms(lambda: audio.logmelfilterbank(wav))
    out["logmel"] = dict(ms=ms, utterances=32, utt_per_s=32 / (ms / 1e3))
    t0 = time.time()
    ref_logmel(wav[0].cpu().numpy())
    out["logmel"]["cpu_oracle_utt_per_s"] = 1.0 / (time.time() - t0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

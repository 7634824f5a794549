"""Batched speech synthesis (generate_speech_batch) on one GPU, Base model in bf16, CUDA-event timed after a warm-up
call that captures the graphs. Steps are fixed by threshold=2.0 (no stop probability reaches it, and the quirk sets
minlenratio = maxlenratio = 2.0: every utterance runs exactly T_enc decoder steps), so the numbers do not depend on an
untrained model's stop flag.
  * TTS: 160-token texts with x-vectors at B = 1, 8, 32;
  * VC: 8 sources of 3 s, then 8 of 30 s, attention record off;
each next to batch-1 generate_speech(use_cache="graph") run B times on the same inputs -> ms per step, utterances / s,
mel frames / s. Also the decode kernel (st5_attn_decode_fwd) alone at the 30 s cross-attention shape (8 x 1 500 keys,
12 heads, bf16): CUDA-event time and bytes / s against the H100 SXM data sheet's 3.35 TB/s, with
bytes = sum_b valid keys x 2 (K, V) x 64 x H x 2 B + q + out.
Prints one JSON line with the card's name and power limit.
usage: python tools/bench_synth_batch.py [--reps 2]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_vc import card  # noqa: E402


def _time(fn, reps):
    import torch
    fn()  # capture / warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1000.0 / reps, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    from speecht5_b200 import ops
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    assert torch.cuda.is_available(), "bench_synth_batch measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    margs = make_args("t5_transformer_base_asr", bert_init=True, build_speech_encoder=True, t5_task="s2s",
                      max_speech_positions=1876)
    model = SpeechT5Task(margs).build_model(margs).to(dev).eval()
    r = model.reduction_factor
    g = torch.Generator().manual_seed(1)
    out = {"metric": "synth_batch", "dtype": "bf16", "threshold": 2.0}

    def row(name, B, batch_fn, one_fn):
        ms, res = _time(batch_fn, args.reps)
        steps = max(m.shape[0] for m, _, _ in res) // r
        frames = sum(m.shape[0] for m, _, _ in res)
        ms1, _ = _time(one_fn, 1)
        out[name] = {"B": B, "steps": steps, "ms": round(ms, 2), "ms_per_step": round(ms / steps, 4),
                     "utt_per_s": round(B * 1000.0 / ms, 2), "frames_per_s": round(frames * 1000.0 / ms, 1),
                     "batch1_x_B_ms": round(ms1, 2), "batch1_ms_per_step": round(ms1 / (B * steps), 4),
                     "speedup": round(ms1 / ms, 2)}

    for B in (1, 8, 32):
        toks = torch.randint(4, 81, (B, 160), generator=g).to(dev)
        spk = torch.randn(B, 512, generator=g).to(dev)
        row(f"tts_160tok_B{B}", B,
            lambda: model.generate_speech_batch(src_tokens=toks, spkembs=spk, threshold=2.0),
            lambda: [model.generate_speech(src_tokens=toks[b:b + 1], spkembs=spk[b:b + 1], threshold=2.0,
                                           use_cache="graph") for b in range(B)])
    for secs, n in ((3, 48_000), (30, 480_256)):
        src = (torch.randn(8, n, generator=g) * 0.1).to(dev)
        pm = torch.zeros_like(src, dtype=torch.bool)
        spk = torch.randn(8, 512, generator=g).to(dev)
        row(f"vc_{secs}s_B8", 8,
            lambda: model.generate_speech_batch(source=src, padding_mask=pm, spkembs=spk, threshold=2.0),
            lambda: [model.generate_speech(source=src[b:b + 1], padding_mask=pm[b:b + 1], spkembs=spk[b:b + 1],
                                           threshold=2.0, use_cache="graph") for b in range(8)])
    # ---- the decode kernel alone at the 30 s cross-attention shape
    B, Tk, H = 8, 1500, 12
    q = torch.randn(B, 1, H * 64, device=dev).to(torch.bfloat16)
    kv = torch.randn(B, Tk, 2 * H * 64, device=dev).to(torch.bfloat16)

    def call():
        return ops.attention_decode(q, kv, H=H, d=H * 64, q_col=0, k_col=0, v_col=1, scale=0.125)
    call()
    torch.cuda.synchronize()
    graph, per_graph, n_replays = torch.cuda.CUDAGraph(), 50, 10  # (replayed: the time is the kernels', not the host's)
    with torch.cuda.graph(graph):
        for _ in range(per_graph):
            call()
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_replays):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    n_calls = per_graph * n_replays
    us = e0.elapsed_time(e1) * 1000.0 / n_calls
    nbytes = B * Tk * 2 * 64 * H * 2 + 2 * B * H * 64 * 2
    out["decode_kernel_30s_cross"] = {"B": B, "Tk": Tk, "H": H, "us": round(us, 2), "bytes": nbytes,
                                      "TB_per_s": round(nbytes / us / 1e6, 3),
                                      "share_of_3.35TB_per_s": round(nbytes / us / 1e6 / 3.35, 3)}
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

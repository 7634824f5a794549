"""Voice conversion (s2s) on one GPU, CUDA-event timed after a warm-up:
  * the fine-tuning update of the VC recipe (SpeechT5 README, voice conversion: t5_transformer_base_asr, guided-attention
    loss, dropout 0.2, encoder LayerDrop 0.05, --max-tokens 1280000 source samples per micro-batch) on 24 pairs of 3.2 s
    sources (51 200 samples) with 200-frame targets and 512-d x-vectors, replayed from one captured CUDA graph by
    B200Trainer in bf16 -> utterances / s;
  * generate_speech of the same model from one 3 s and one 30 s source (use_cache "graph", the defaults of
    scripts/generate_speech.py: threshold 0.5, maxlenratio 10) in bf16 -> ms per utterance, decoder steps, ms per step,
    the graph cache the synthesis keeps on the model (its buffers are sized by the step budget T_enc * 10 / 2, not by
    the steps taken) and the peak above the resident model, cache included. The model is untrained: its stop flag
    fires after the number of steps printed, far below the budget, so the per-step times are those of short decodes.
Prints one JSON line with the card's name and power limit beside the numbers.
usage: python tools/bench_vc.py [--steps 20] [--warmup 5] [--reps 2]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECIPE = dict(dropout=0.2, activation_dropout=0.2, attention_dropout=0.2, encoder_layerdrop=0.05, decoder_layerdrop=0.0,
              feature_grad_mult=1.0, bert_init=True, relative_position_embedding=True, mask_prob=0.0,
              mask_channel_prob=0.0, max_speech_positions=1876, build_speech_encoder=True, t5_task="s2s")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2, help="timed generate_speech calls per source length")
    ap.add_argument("--batch", type=int, default=24)
    args = ap.parse_args()
    import torch
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_vc_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    assert torch.cuda.is_available(), "bench_vc measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    margs = make_args("t5_transformer_base_asr", **RECIPE)
    task = SpeechT5Task(margs)
    model = task.build_model(margs).to(dev).train()
    crit = SpeechT5Criterion(task, use_guided_attn_loss=True)
    trainer = B200Trainer(model, crit, task, lr=1e-4)
    sample = synthetic_vc_batch(args.batch, 51200, 200, seed=1, ragged=False, pin=True)
    for _ in range(args.warmup):
        trainer.train_step([sample])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        losses, stats = trainer.train_step([sample])
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps
    assert bool(torch.isfinite(losses).all()), "non-finite loss"
    out = {"metric": "s2s_update_utt_per_s", "update_ms": round(step_ms, 3),
           "utt_per_s": round(args.batch * 1000.0 / step_ms, 1), "batch": args.batch, "source_samples": 51200,
           "target_frames": 200, "graph_hits": trainer.graph_hits, "graph_misses": trainer.graph_misses}
    del trainer, losses, stats
    # ---- generate_speech from one source of 3 s and one of 30 s
    model.eval()
    g = torch.Generator().manual_seed(2)
    spk = torch.randn(1, 512, generator=g).to(dev)
    for secs, n in ((3, 48_000), (30, 480_256)):
        source = (torch.randn(1, n, generator=g) * 0.1).to(dev)
        pm = torch.zeros_like(source, dtype=torch.bool)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        mel, _, attn = model.generate_speech(source=source, padding_mask=pm, spkembs=spk, use_cache="graph")  # capture
        torch.cuda.synchronize()
        cache = torch.cuda.memory_allocated() - base  # the bucket's SynthesisGraph buffers, kept on the model
        e0.record()
        for _ in range(args.reps):
            mel, _, attn = model.generate_speech(source=source, padding_mask=pm, spkembs=spk, use_cache="graph")
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        steps = mel.shape[0] // model.reduction_factor
        out.update({f"synth_{secs}s_ms": round(ms, 2), f"synth_{secs}s_steps": steps,
                    f"synth_{secs}s_enc_frames": attn.shape[-1], f"synth_{secs}s_ms_per_step": round(ms / steps, 4),
                    f"synth_{secs}s_graph_cache_gib": round(cache / 2 ** 30, 3),
                    f"synth_{secs}s_peak_extra_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)})
    out.update({"card": card(), "dtype": "bf16"})
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Speaker identification (s2c) on one GPU, CUDA-event timed after a warm-up:
  * the fine-tuning update of the recipe (SpeechT5 README, speaker identification: t5_transformer_base_asr, softmax head
    on the pooled decoder state, no pooling BN, no embedding post-net, dropout 0.1, encoder LayerDrop 0.05) on 8
    crops of 3.2 s (51 200 samples, the training crop of tasks/speecht5.py:379) over 1 255 classes, replayed from one
    captured CUDA graph by B200Trainer in bf16 -> utterances / s;
  * generate_class of the same model on ONE 160 s utterance (2 560 000 samples, 7 999 encoder frames; test utterances
    are not cropped, tasks/speecht5.py:383) in bf16 -> latency and peak memory.
Prints one JSON line with the card's name and power limit beside the numbers.
usage: python tools/bench_sid.py [--steps 20] [--warmup 5] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECIPE = dict(dropout=0.1, activation_dropout=0.1, attention_dropout=0.1, encoder_layerdrop=0.05, decoder_layerdrop=0.0,
              feature_grad_mult=1.0, bert_init=True, relative_position_embedding=True, share_input_output_embed=True,
              mask_prob=0.0, mask_channel_prob=0.0, sid_no_pooling_bn=True, sid_no_embed_postnet=True,
              max_text_positions=600, max_speech_positions=8000, build_speech_encoder=True, build_text_decoder=True,
              t5_task="s2c", vocab_size=1255)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="timed generate_class calls")
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    import torch
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_sid_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    assert torch.cuda.is_available(), "bench_sid measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    margs = make_args("t5_transformer_base_asr", **RECIPE)
    task = SpeechT5Task(margs)
    model = task.build_model(margs).to(dev).train()
    crit = SpeechT5Criterion(task, label_smoothing=0.1, report_accuracy=True)
    trainer = B200Trainer(model, crit, task, lr=2e-4, weight_decay=0.1)
    sample = synthetic_sid_batch(args.batch, 51200, 1255, seed=1, ragged=False, pin=True)
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
    out = {"metric": "s2c_update_utt_per_s", "update_ms": round(step_ms, 3),
           "utt_per_s": round(args.batch * 1000.0 / step_ms, 1), "batch": args.batch, "crop_samples": 51200,
           "classes": 1255, "graph_hits": trainer.graph_hits, "graph_misses": trainer.graph_misses}
    del trainer, losses, stats
    # ---- generate_class on one 160 s utterance
    model.eval()
    g = torch.Generator().manual_seed(2)
    source = (torch.randn(1, 2_560_000, generator=g) * 0.1).to(dev)
    pm = torch.zeros_like(source, dtype=torch.bool)
    prev = torch.full((1, 1), 2, dtype=torch.long, device=dev)
    pred = model.generate_class(source, prev, padding_mask=pm)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0.record()
    for _ in range(args.reps):
        pred = model.generate_class(source, prev, padding_mask=pm)
    e1.record()
    torch.cuda.synchronize()
    out.update({"generate_class_160s_ms": round(e0.elapsed_time(e1) / args.reps, 2),
                "generate_class_peak_extra_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3),
                "predicted": int(pred[0]), "card": card(), "dtype": "bf16"})
    print(json.dumps(out))


if __name__ == "__main__":
    main()

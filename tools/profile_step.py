"""Where the GPU time of one TTS fine-tune update goes, per kernel, from torch.profiler (CUDA activities).

Builds the model, batch and seeds of bench.py's tts workload, runs two eager warm-up updates and then one eager update
under the profiler. Writes OUT/kernels.json and OUT/kernels.txt: every device activity (kernels, copies, sets) summed
per name -- launches and total microseconds -- sorted by time, plus the busy total of the update.

  python tools/profile_step.py --out DIR [--batch 32]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.autograd import DeviceType  # noqa: E402

from bench import WORKLOAD  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=WORKLOAD["batch_per_gpu"])
    args = ap.parse_args()
    from speecht5_b200 import _lib
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_tts_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer, _to_device
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib = _lib.load()
    _lib.check(lib.st5_device_ok(), "st5_device_ok")
    RT.dtype = torch.bfloat16
    RT.manual_seed(1)
    torch.manual_seed(1337)
    margs = make_args(WORKLOAD["arch"], encoder_layerdrop=0.0, decoder_layerdrop=0.0, bert_init=True,
                      decoder_layers=WORKLOAD["decoder_layers"], share_input_output_embed=True, max_text_positions=600,
                      max_speech_positions=1876)
    task = SpeechT5Task(margs)
    model = task.build_model(margs).to(dev).train()
    crit = SpeechT5Criterion(task, use_guided_attn_loss=True)
    trainer = B200Trainer(model, crit, task, lr=1e-4, betas=(0.9, 0.98), eps=1e-8, clip_norm=25.0,
                          use_cuda_graph=False)
    batches = [_to_device(synthetic_tts_batch(args.batch, WORKLOAD["text_len"], WORKLOAD["mel_frames"], seed=i), dev)
               for i in range(3)]
    for i in range(2):
        trainer.train_step([batches[i]])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        trainer.train_step([batches[2]])
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0, 0.0])
    t0, t1 = None, None
    for e in prof.profiler.kineto_results.events():
        if e.device_type() != DeviceType.CUDA:
            continue
        s = per[e.name()]
        s[0] += 1
        s[1] += e.duration_ns() * 1e-3
        t0 = e.start_ns() if t0 is None else min(t0, e.start_ns())
        t1 = e.end_ns() if t1 is None else max(t1, e.end_ns())
    rows = sorted(({"name": k, "launches": v[0], "total_us": round(v[1], 1)} for k, v in per.items()),
                  key=lambda r: -r["total_us"])
    busy = sum(r["total_us"] for r in rows)
    span = (t1 - t0) * 1e-3 if t0 is not None else 0.0
    os.makedirs(args.out, exist_ok=True)
    summary = dict(gpu=torch.cuda.get_device_name(dev), batch=args.batch, busy_us=round(busy, 1),
                   span_us=round(span, 1), kernels=rows)
    with open(os.path.join(args.out, "kernels.json"), "w") as fh:
        json.dump(summary, fh, indent=1)
    with open(os.path.join(args.out, "kernels.txt"), "w") as fh:
        fh.write(f"{summary['gpu']}  batch {args.batch}  busy {busy:.1f} us  span {span:.1f} us\n")
        for r in rows:
            fh.write(f"{r['total_us']:>10.1f} us {r['launches']:>5d}  {r['name'][:160]}\n")
    print(open(os.path.join(args.out, "kernels.txt")).read()[:4000])


if __name__ == "__main__":
    main()

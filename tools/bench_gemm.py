"""Where the GEMM time of the TTS fine-tune update goes, per launch class, on one GPU.

Builds the model and trainer of `bench.py` (tts workload: SpeechT5-Base, 32 x 10 s utterances, bf16), records the
st5_gemm_bf16 launches of one eager update and groups them by (M, N, K, batch, tile width, epilogue). Each class is
replayed inside a captured CUDA graph and timed with CUDA events: launches per update, ms per update, TFLOP/s, tiles per
CTA. The epilogue proxy is the same launches with K cut to one k-block (64): per tile that is the epilogue plus one
k-block of MMAs, so proxy / full estimates the share of the class's time spent outside the main loop when nothing
overlaps it. The card's name, power limit and maximum SM clock are read (read-only) with nvidia-smi.
usage: python tools/bench_gemm.py [--reps 20] [--batch 32] [--json PATH]"""
import argparse
import collections
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ACT_NAMES = {0: "", 1: "relu", 2: "gelu", 3: "tanh", 4: "gelu_tanh", 5: "gate", 6: "gelu_tanh_gate"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def tile_width(g, sms):
    """The tile width gemm_launch's cost model picks (csrc/gemm.cu), unless ST5_GEMM_BN pins it."""
    force = int(os.environ.get("ST5_GEMM_BN", "0") or 0)
    if force in (64, 128):
        return force
    tiles_m = -(-g.M // 128)
    batch = g.nb1 * g.nb2

    def cost(bn, factor):
        rounds = -(-(tiles_m * -(-g.N // bn) * batch) // sms)
        return rounds * (bn * factor + 24.0)
    c128 = cost(128, 1.0) if g.N > 64 else 1e30
    return 128 if c128 <= cost(64, 1.25) else 64


def epilogue_kind(g):
    parts = []
    if g.act == 6:
        parts.append("gate")
    elif g.act:
        parts.append(ACT_NAMES[g.act])
    if g.bias:
        parts.append("bias")
    if g.bias2:
        parts.append("bias2")
    if g.c_pre and g.act != 6:
        parts.append("pre")
    if g.drop_p > 0:
        parts.append("dropout")
    if g.residual:
        parts.append("residual")
    if g.actgrad_pre:
        parts.append("x" + ACT_NAMES[g.actgrad_act] + "'")
    if g.accumulate:
        parts.append(f"acc{g.accumulate}")
    if g.alpha != 1.0:
        parts.append("alpha")
    parts.append("f32" if g.c_fp32 else "bf16")
    return "+".join(parts) if len(parts) > 1 else "plain+" + parts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="graph replays per timed class")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    args = ap.parse_args()
    import torch
    from bench import WORKLOAD
    from speecht5_b200 import _lib
    from speecht5_b200 import kernels as K
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_tts_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer, _to_device
    assert torch.cuda.is_available(), "bench_gemm measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _lib.load()
    _lib.check(lib.st5_device_ok(), "st5_device_ok")
    RT.dtype = torch.bfloat16
    RT.manual_seed(1)
    torch.manual_seed(1337)
    margs = make_args(WORKLOAD["arch"], encoder_layerdrop=0.0, decoder_layerdrop=0.0, bert_init=True,
                      decoder_layers=WORKLOAD["decoder_layers"], share_input_output_embed=True,
                      max_text_positions=600, max_speech_positions=1876)
    task = SpeechT5Task(margs)
    model = task.build_model(margs).to(dev).train()
    trainer = B200Trainer(model, SpeechT5Criterion(task, use_guided_attn_loss=True), task, lr=1e-4,
                          betas=(0.9, 0.98), eps=1e-8, clip_norm=25.0, use_cuda_graph=False)
    batches = [_to_device(synthetic_tts_batch(args.batch, WORKLOAD["text_len"], WORKLOAD["mel_frames"], seed=i), dev)
               for i in range(3)]
    for b in batches[:2]:
        trainer.train_step([b])
    torch.cuda.synchronize()
    K.GEMM_RECORD = []
    trainer.train_step([batches[2]])
    torch.cuda.synchronize()
    records, K.GEMM_RECORD = K.GEMM_RECORD, None

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    classes = collections.OrderedDict()
    for g in records:
        key = (g.M, g.N, g.K, g.nb1 * g.nb2, tile_width(g, sms), epilogue_kind(g))
        classes.setdefault(key, []).append(g)

    def time_launches(launches):
        K.gemm_replay(launches)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            K.gemm_replay(launches)
        graph.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    rows = []
    for (M, N, Kd, nb, bn, kind), launches in classes.items():
        proxies = []
        for g in launches:
            c = type(g).from_buffer_copy(g)
            c.K = min(Kd, 64)
            proxies.append(c)
        flop = 2.0 * M * N * Kd * nb * len(launches)
        ms = time_launches(launches)
        ms_proxy = time_launches(proxies)
        tiles = -(-M // 128) * -(-N // bn) * nb
        rows.append(dict(M=M, N=N, K=Kd, batch=nb, bn=bn, epilogue=kind, launches=len(launches), ms=ms,
                         tflops=flop / (ms * 1e-3) / 1e12, tiles_per_cta=tiles / min(tiles, sms), proxy_ms=ms_proxy,
                         proxy_share=ms_proxy / ms))
    total = sum(r["ms"] for r in rows)
    total_flop = sum(2.0 * g.M * g.N * g.K * g.nb1 * g.nb2 for g in records)
    print(f"card: {card()}  (name, power.limit, clocks.max.sm)")
    print(f"{len(records)} GEMM launches in {len(rows)} classes, {total_flop / 1e12:.2f} TFLOP per update, "
          f"{total:.2f} ms summed over classes ({total_flop / (total * 1e-3) / 1e12:.0f} TFLOP/s)")
    hdr = f"{'M':>6} {'N':>5} {'K':>5} {'nb':>3} {'BN':>3} {'epilogue':<34} {'n':>3} {'ms/upd':>7} {'share':>6} " \
          f"{'TFLOP/s':>7} {'t/CTA':>6} {'proxy ms':>8} {'proxy/full':>10}"
    print(hdr)
    for r in sorted(rows, key=lambda r: -r["ms"]):
        print(f"{r['M']:>6} {r['N']:>5} {r['K']:>5} {r['batch']:>3} {r['bn']:>3} {r['epilogue']:<34} "
              f"{r['launches']:>3} {r['ms']:>7.3f} {r['ms'] / total:>6.1%} {r['tflops']:>7.0f} "
              f"{r['tiles_per_cta']:>6.1f} {r['proxy_ms']:>8.3f} {r['proxy_share']:>10.2f}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=card(), total_ms=total, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()

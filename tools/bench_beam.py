"""Beam search for text output on the GPU: T5TransformerModel.generate_text_beam(use_cache="graph") on Base
(t5_transformer_base_asr, bf16, random weights), 8 utterances of 10 s and one of 10 s alone, beam 5 and 10, next to the
beam-1 GreedyGraph on the same inputs. The number of steps is fixed with min_len = max_len (eos is banned until the last
step, where it is the only choice), so an untrained model's outputs do not change the timing. Encoder included.

With --lm, the same beam rows again with LM shallow fusion (`lm=`, `lm_weight` 0.5): a random-weight fairseq
transformer_lm of base size (6 layers x 512, 8 heads, FFN 2048, vocabulary V - 2) run inside every captured step, or with
--lm-arch transformer_lm_t5 SpeechT5's own LM (20 layers x 1280, 16 heads of 80, FFN 6144, GELU); with it, the LM's
key/value cache per bucket, the peak memory a beam decode allocates above the resident models, and the 80-wide
st5_attn_lineage_hd_fwd alone at its full-size shape (8 sentences x K beams, 16 heads, a lineage table over 256 cached
positions) with bytes per second from shapes.

Also CUDA-event times of st5_beam_topk (and, with --lm, st5_beam_topk_lm at V_lm = V - 2) and st5_beam_update alone (V = 81 and V = 8 000, the ASR character and the
MuST-C ST vocabularies) and of st5_attn_lineage_fwd at the 10 s cross-attention shape (8 sentences x K beams over one
copy of 500 encoder keys per sentence, 12 heads), with bytes per second from shapes.
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import subprocess


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


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64, help="decoder steps per decode (min_len = max_len)")
    ap.add_argument("--lm", action="store_true", help="also the LM-fusion rows")
    ap.add_argument("--lm-arch", default="transformer_lm", choices=("transformer_lm", "transformer_lm_t5"),
                    help="the LM of the --lm rows: base transformer_lm (6 x 512) or transformer_lm_t5 (20 x 1280)")
    args = ap.parse_args()
    import torch
    from speecht5_b200 import kernels
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    if not torch.cuda.is_available():
        raise SystemExit("bench_beam.py measures on a CUDA device; none found")
    dev = torch.device("cuda", 0)
    RT.dtype = torch.bfloat16
    torch.manual_seed(0)
    name, power = card()
    out = {"card": name, "power_limit": power, "steps": args.steps}
    margs = make_args("t5_transformer_base_asr", build_speech_encoder=True, build_text_decoder=True, bert_init=True,
                      encoder_layerdrop=0.0, decoder_layerdrop=0.0, max_text_positions=600)
    asr = T5TransformerModel.build_model(margs).to(dev).eval()
    wav = torch.randn(8, 160000, device=dev) * 0.1
    wpm = torch.zeros(8, 160000, dtype=torch.bool, device=dev)
    n = args.steps
    kw = dict(max_len_b=n, min_len=n)
    ms = cuda_ms(lambda: asr.generate_text_greedy(wav, wpm, use_cache="graph", **kw))
    out["greedy_graph_B8"] = dict(ms=ms, ms_per_step=ms / (n + 1), utt_per_s=8 / (ms / 1e3))
    for K in (5, 10):
        ms8 = cuda_ms(lambda: asr.generate_text_beam(wav, wpm, beam_size=K, use_cache="graph", **kw))
        ms1 = cuda_ms(lambda: asr.generate_text_beam(wav[:1], wpm[:1], beam_size=K, use_cache="graph", **kw))
        out[f"beam{K}_graph"] = dict(ms_B8=ms8, ms_per_step_B8=ms8 / (n + 1), utt_per_s_B8=8 / (ms8 / 1e3), ms_B1=ms1,
                                     ms_per_step_B1=ms1 / (n + 1), speedup_B8_over_8x_B1=8 * ms1 / ms8)
    if args.lm:
        from argparse import Namespace
        from speecht5_b200.lm import TransformerLM
        V = asr.text_decoder_postnet.output_projection.weight.shape[0]
        if args.lm_arch == "transformer_lm_t5":
            lm = TransformerLM(Namespace(arch="transformer_lm_t5"), V - 2)
        else:
            lm = TransformerLM(Namespace(decoder_layers=6, decoder_embed_dim=512, decoder_attention_heads=8,
                                         decoder_ffn_embed_dim=2048), V - 2)
        for p in lm.parameters():
            torch.nn.init.normal_(p, std=0.05)
        lm = lm.to(dev)
        out["lm_arch"] = args.lm_arch
        for K in (5, 10):
            torch.cuda.synchronize()
            resident = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            ms8 = cuda_ms(lambda: asr.generate_text_beam(wav, wpm, beam_size=K, use_cache="graph", lm=lm, lm_weight=0.5,
                                                         **kw))
            row = dict(ms_B8=ms8, ms_per_step_B8=ms8 / (n + 1), utt_per_s_B8=8 / (ms8 / 1e3))
            if args.lm_arch == "transformer_lm_t5":
                bg = [g for key, g in asr.__dict__.get("_beam_graphs", {}).items() if key[1] == K and g.lm is lm]
                row["lm_cache_MiB"] = sum(c.numel() * c.element_size() for c in bg[0].lm_cache.self_kv) / 2 ** 20
                row["peak_above_resident_MiB"] = (torch.cuda.max_memory_allocated() - resident) / 2 ** 20
            out[f"beam{K}_lm_graph"] = row
    del asr
    # kernels alone
    B, t = 8, torch.tensor([5], dtype=torch.int64, device=dev)
    mn, mx = torch.tensor([1], dtype=torch.int64, device=dev), torch.tensor([100], dtype=torch.int64, device=dev)
    for V in (81, 8000):
        for K in (5, 10):
            logits = torch.randn(B * K, V, device=dev).to(torch.bfloat16)
            cum, mask = -torch.rand(B * K, device=dev), torch.zeros(V, device=dev)
            cs = torch.empty(B, 2 * K, device=dev)
            ct, cb = (torch.empty(B, 2 * K, dtype=torch.int32, device=dev) for _ in range(2))
            us = 1e3 * cuda_ms(lambda: kernels.beam_topk(logits, cum, mask, 1.0, 2, t, mn, mx, cs, ct, cb, K=K), reps=200)
            out[f"beam_topk_V{V}_K{K}_us"] = us
            if args.lm:
                lm_logits = torch.randn(B * K, V - 2, device=dev)
                us = 1e3 * cuda_ms(lambda: kernels.beam_topk(logits, cum, mask, 1.0, 2, t, mn, mx, cs, ct, cb, K=K,
                                                             lm_logits=lm_logits, lm_weight=0.5), reps=200)
                out[f"beam_topk_lm_V{V}_K{K}_us"] = us
    for K in (5, 10):
        T = 73
        i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
        st = dict(t=torch.zeros(1, dtype=torch.int64, device=dev), max_len=torch.zeros(1, dtype=torch.int64, device=dev),
                  cand_score=torch.zeros((B, 2 * K), **f32), cand_token=torch.zeros((B, 2 * K), **i32),
                  cand_beam=torch.zeros((B, 2 * K), **i32), lin=torch.zeros((B * K, T), **i32),
                  tok=torch.zeros((B * K, T), **i32), score=torch.zeros((B * K, T), **f32),
                  ignore=torch.zeros(B * K, **i32), finished=torch.zeros(B, **i32), parent=torch.zeros(B * K, **i32),
                  cur_tok=torch.zeros(B * K, dtype=torch.int64, device=dev), cur_score=torch.zeros(B * K, **f32),
                  fin_n=torch.zeros(B, **i32), fin_tok=torch.zeros((B, K, T), **i32),
                  fin_pos=torch.zeros((B, K, T), **f32), fin_len=torch.zeros((B, K), **i32),
                  fin_score=torch.zeros((B, K), **f32), stop=torch.zeros(T, **i32))
        st["t"].fill_(5)
        st["max_len"].fill_(64)
        st["cand_token"].fill_(7)
        st["cand_score"].copy_(-torch.arange(2 * K, device=dev).float().expand(B, 2 * K))

        def upd():
            st["finished"].zero_()
            kernels.beam_update(st, K=K, V=8000, eos=2, normalize=True, len_penalty=1.0)
        out[f"beam_update_K{K}_us"] = 1e3 * cuda_ms(upd, reps=200)
    H, S = 12, 500
    for K in (5, 10):
        q = torch.randn(B * K, 1, H * 64, device=dev).to(torch.bfloat16)
        kv = torch.randn(B, S, 2 * H * 64, device=dev).to(torch.bfloat16)
        o = torch.empty(B * K, 1, H * 64, device=dev, dtype=torch.bfloat16)
        pad = torch.zeros(B * K, S, dtype=torch.uint8, device=dev)
        us = 1e3 * cuda_ms(lambda: kernels.attn_lineage_fwd(q, kv[:, :, :H * 64], kv[:, :, H * 64:], o, H=H, scale=0.125,
                                                             key_pad=pad, kv_div=K), reps=200)
        # each query row reads its sentence's keys and values (L2 serves the K-fold reuse; this counts what is read)
        nbytes = B * K * S * 2 * H * 64 * 2 + q.numel() * 2 * 2 + pad.numel()
        out[f"attn_lineage_cross_K{K}"] = dict(us=us, GBps=nbytes / (us * 1e-6) / 1e9)
    if args.lm and args.lm_arch == "transformer_lm_t5":
        H, hd, T = 16, 80, 256  # (transformer_lm_t5's self-attention: 16 heads of 80, 256 cached positions)
        for K in (5, 10):
            BK, rows = B * K, T + 9
            q = torch.randn(BK, 1, 3 * H * hd, device=dev).to(torch.bfloat16)
            cache = torch.randn(BK, rows, 2 * H * hd, device=dev).to(torch.bfloat16)
            o = torch.empty(BK, 1, H * hd, device=dev, dtype=torch.bfloat16)
            pad = torch.zeros(BK, T, dtype=torch.uint8, device=dev)
            # a lineage table as beam reorders leave it: each position from some beam row of the same sentence
            lin = (torch.arange(BK, device=dev)[:, None] // K * K
                   + torch.randint(0, K, (BK, rows), device=dev)).to(torch.int32)
            us = 1e3 * cuda_ms(lambda: kernels.attn_lineage_hd_fwd(
                q[:, :, :H * hd], cache[:, :T, :H * hd], cache[:, :T, H * hd:], o, H=H, head_dim=hd, scale=hd ** -0.5,
                key_pad=pad, kv_rows=lin), reps=200)
            nbytes = BK * T * 2 * H * hd * 2 + BK * H * hd * 2 * 2 + pad.numel() + BK * T * 4
            out[f"attn_lineage_hd80_self_K{K}_T{T}"] = dict(us=us, GBps=nbytes / (us * 1e-6) / 1e9)
    print(json.dumps(out))


if __name__ == "__main__":
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    main()

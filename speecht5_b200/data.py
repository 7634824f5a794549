"""Synthetic batches with the reference collaters' key contract (host I/O itself -- soundfile, librosa log-mel,
manifests -- is outside the hot path). TTS: speecht5/data/text_to_speech_dataset.py:223-281 (right-padded text tokens,
mel targets [B, L, 80], prev_output_tokens = [0; every r-th frame][:-1], stop labels 1 from the last real frame on,
512-d x-vectors)."""
import torch


def synthetic_tts_batch(B, T_txt, T_mel, vocab=81, odim=80, r=2, seed=1, ragged=True, pad=1, pin=False):
    g = torch.Generator().manual_seed(seed)
    src_lengths = (torch.randint(int(0.75 * T_txt), T_txt + 1, (B,), generator=g) if ragged and B > 1
                   else torch.full((B,), T_txt))
    src_lengths[0] = T_txt
    src_tokens = torch.randint(4, vocab, (B, T_txt), generator=g)
    ar = torch.arange(T_txt)[None, :]
    src_tokens = torch.where(ar < src_lengths[:, None], src_tokens, torch.full_like(src_tokens, pad))
    mel_lengths = (torch.randint(int(0.9 * T_mel), T_mel + 1, (B,), generator=g) if ragged and B > 1
                   else torch.full((B,), T_mel))
    mel_lengths[0] = T_mel
    fbank = torch.randn(B, T_mel, odim, generator=g)
    am = torch.arange(T_mel)[None, :]
    fbank = fbank * (am < mel_lengths[:, None]).unsqueeze(-1)
    fb_in = fbank[:, r - 1::r]
    len_in = torch.div(mel_lengths, r, rounding_mode="floor")
    prev = torch.cat([fb_in.new_zeros((B, 1, odim)), fb_in[:, :-1]], dim=1).contiguous()
    labels = (am >= (mel_lengths[:, None] - 1)).float()
    spk = torch.randn(B, 512, generator=g)
    net_input = dict(src_tokens=src_tokens, src_lengths=src_lengths, prev_output_tokens=prev, tgt_lengths=len_in,
                     spkembs=spk, task_name="t2s")
    sample = dict(net_input=net_input, labels=labels, dec_target=fbank, dec_target_lengths=mel_lengths,
                  src_lengths=src_lengths, task_name="t2s", ntokens=int(src_lengths.sum()), target=fbank)
    if pin:
        sample = _pin(sample)
    return sample


def synthetic_asr_batch(B, n_samples, T_tgt, vocab=81, seed=1, ragged=True, pin=False):
    """SURVEY 8(d) config 3 shaped batch through the s2t collater: waveforms N(0, 0.1^2) with lengths U{0.8 n .. n}
    (-> padding_mask), `T_tgt - 1` target tokens U{4 .. vocab-3} + eos (the last two ids are <mask> / <ctc_blank>,
    tasks/speecht5.py:283-287)."""
    g = torch.Generator().manual_seed(seed)
    items = []
    for b in range(B):
        n = n_samples if (b == 0 or not ragged) else int(torch.randint(int(0.8 * n_samples), n_samples + 1, (1,), generator=g))
        t = T_tgt - 1 if (b == 0 or not ragged) else int(torch.randint(max(1, T_tgt // 2), T_tgt, (1,), generator=g))
        items.append({"id": b, "source": torch.randn(n, generator=g) * 0.1,
                      "label_list": [torch.randint(4, vocab - 2, (t,), generator=g)]})
    sample = collate_asr(items)
    return _pin(sample) if pin else sample


def synthetic_speech_pretrain_batch(B, n_samples, n_classes=500, label_rate=50, sample_rate=16000, hop=256, odim=80, r=2,
                                    seed=1, pin=False):
    """SURVEY 8(d) config 4, speech micro-batch, with the key contract of speecht5/data/speech_dataset.py:302-386 for the
    pre-training recipe (pad_audio False: every waveform cropped to one length, so the padding mask is all False):
    waveforms N(0, 0.1^2) [B, n], HuBERT k-means labels U{0..n_classes-1} at `label_rate` Hz (:409-425: round(n *
    rate / 16000) per utterance), log-mel reconstruction target [B, 1 + n // hop, odim], decoder input = every r-th
    frame shifted by one (:335-344), stop labels 1 from the last real frame on (:346-349), 512-d x-vectors."""
    g = torch.Generator().manual_seed(seed)
    wave = torch.randn(B, n_samples, generator=g) * 0.1
    L = 1 + n_samples // hop
    fbank = torch.randn(B, L, odim, generator=g)
    fb_in = fbank[:, r - 1::r]
    len_in = torch.full((B,), L // r, dtype=torch.long)
    prev = torch.cat([fb_in.new_zeros((B, 1, odim)), fb_in[:, :-1]], dim=1).contiguous()
    labels = torch.zeros(B, L)
    labels[:, L - 1:] = 1.0
    n_lab = int(round(n_samples * label_rate / sample_rate))
    km = torch.randint(0, n_classes, (B, n_lab), generator=g)
    net_input = dict(source=wave, padding_mask=torch.zeros(B, n_samples, dtype=torch.bool), prev_output_tokens=prev,
                     spkembs=torch.randn(B, 512, generator=g), tgt_lengths=len_in)
    sample = dict(id=torch.arange(B), net_input=net_input, labels=labels, dec_target=fbank,
                  dec_target_lengths=torch.full((B,), L, dtype=torch.long), src_lengths=[n_samples] * B,
                  task_name="speech_pretrain", target_lengths_list=[torch.full((B,), n_lab, dtype=torch.long)],
                  ntokens_list=[B * n_lab], target_list=[km])
    return _pin(sample) if pin else sample


def synthetic_text_pretrain_batch(B, T, vocab, mask_idx, mask_ratio=0.3, pad=1, eos=2, seed=1, pin=False):
    """SURVEY 8(d) config 4, text micro-batch: `--sample-break-mode eos --tokens-per-sample 512` blocks through the
    denoising collater (speecht5/data/text_dataset.py:18-98 `collate`, called from :434-443: source = noised tokens, target = the
    clean block, prev_output_tokens = the target rotated so that eos comes first). The BART span infilling itself is the
    host pipeline's; here `mask_ratio` of the positions carry <mask> (same shapes: the step's cost does not depend on
    which positions)."""
    g = torch.Generator().manual_seed(seed)
    target = torch.randint(4, vocab - 2, (B, T), generator=g)
    target[:, -1] = eos
    source = target.clone()
    hide = torch.rand(B, T - 1, generator=g) < mask_ratio
    source[:, :-1][hide] = mask_idx
    prev = torch.cat([target[:, -1:], target[:, :-1]], dim=1).contiguous()
    sample = dict(id=torch.arange(B), nsentences=B, ntokens=B * T, target=target, task_name="text_pretrain",
                  net_input=dict(src_tokens=source, src_lengths=torch.full((B,), T, dtype=torch.long),
                                 prev_output_tokens=prev))
    return _pin(sample) if pin else sample


def collate_frames(frames, is_audio_input=False):
    """text_to_speech_dataset.py:25-45 _collate_frames: zero-padded stack of [L_i, F] (or [L_i]) tensors."""
    max_len = max(f.size(0) for f in frames)
    shape = (len(frames), max_len) if is_audio_input else (len(frames), max_len, frames[0].size(1))
    out = frames[0].new_zeros(shape)
    for i, v in enumerate(frames):
        out[i, : v.size(0)] = v
    return out


def collate_tts(samples, reduction_factor=2, pad=1):
    """TextToSpeechDataset.collater (text_to_speech_dataset.py:226-281) over in-memory items
    {"id", "source": [LongTensor tokens], "target": FloatTensor [L, odim], "spkembs": FloatTensor [512],
    "audio_name"}: the batch dict the task, the criterion and the trainer consume. Host-side work only."""
    samples = [s for s in samples if s["source"] is not None]
    if len(samples) == 0:
        return {}
    fbanks = [s["target"] for s in samples]
    fbank_sizes = [len(f) for f in fbanks]
    collated = collate_frames(fbanks)
    sizes = torch.tensor(fbank_sizes, dtype=torch.long)
    r = reduction_factor
    if r > 1:  # thin out frames for the reduction factor: (B, Lmax, odim) -> (B, Lmax // r, odim)
        fb_in = collated[:, r - 1::r]
        sizes_in = torch.div(sizes, r, rounding_mode="floor")
    else:
        fb_in, sizes_in = collated, sizes
    prev = torch.cat([fb_in.new_zeros((fb_in.shape[0], 1, fb_in.shape[2])), fb_in[:, :-1]], dim=1)
    labels = collated.new_zeros(collated.size(0), collated.size(1))
    for i, n in enumerate(fbank_sizes):
        labels[i, n - 1:] = 1.0
    spkembs = collate_frames([s["spkembs"] for s in samples], is_audio_input=True)
    toks = [s["source"][0] for s in samples]
    lengths = torch.LongTensor([len(t) for t in toks])
    src = toks[0].new_full((len(toks), int(lengths.max())), pad)  # data_utils.collate_tokens(left_pad=False)
    for i, t in enumerate(toks):
        src[i, : len(t)] = t
    net_input = {"src_tokens": src, "src_lengths": lengths, "prev_output_tokens": prev, "tgt_lengths": sizes_in,
                 "spkembs": spkembs, "task_name": "t2s"}
    return {"id": torch.LongTensor([s["id"] for s in samples]), "name": [s.get("audio_name") for s in samples],
            "net_input": net_input, "labels": labels, "dec_target": collated, "dec_target_lengths": sizes,
            "src_lengths": lengths, "task_name": "t2s", "ntokens": int(lengths.sum().item()), "target": collated}


def collate_asr(samples, pad=1, eos=2):
    """SpeechToTextDataset.collater (speecht5/data/speech_to_text_dataset.py:150-222) over in-memory items
    {"id", "source": FloatTensor [N] waveform, "label_list": [LongTensor tokens]}: zero-padded waveforms with their
    boolean padding mask, targets = tokens + eos (right padded), prev_output_tokens = the same with eos moved to the
    front (fairseq collate_tokens(move_eos_to_beginning=True)). Host-side work only."""
    samples = [s for s in samples if s["source"] is not None]
    if len(samples) == 0:
        return {}
    source, padding_mask = _collate_audio([s["source"] for s in samples])
    labels = [torch.cat((s["label_list"][0].long(), torch.tensor([eos]))) for s in samples]
    lengths = torch.tensor([len(t) for t in labels], dtype=torch.long)
    T = int(lengths.max())
    target = torch.full((len(labels), T), pad, dtype=torch.long)
    prev = torch.full((len(labels), T), pad, dtype=torch.long)
    for i, t in enumerate(labels):
        target[i, : len(t)] = t
        prev[i, 0] = eos
        prev[i, 1: len(t)] = t[:-1]
    ntokens = int(sum(len(s["label_list"][0]) for s in samples))
    return {"id": torch.LongTensor([s["id"] for s in samples]),
            "net_input": {"source": source, "padding_mask": padding_mask, "prev_output_tokens": prev,
                          "task_name": "s2t"},
            "target": target, "target_lengths": lengths, "task_name": "s2t", "ntokens": ntokens}


def _collate_audio(audios):
    """Zero-padded waveforms [B, n_max] and their boolean padding mask (True on padding)."""
    n = max(len(a) for a in audios)
    source = audios[0].new_zeros(len(audios), n)
    padding_mask = torch.zeros(len(audios), n, dtype=torch.bool)
    for i, a in enumerate(audios):
        source[i, : len(a)] = a
        padding_mask[i, len(a):] = True
    return source, padding_mask


def collate_sid(samples, pad=1, eos=2):
    """SpeechToClassDataset.collater (speecht5/data/speech_to_class_dataset.py:138-198) over in-memory items
    {"id", "source": FloatTensor [N] waveform, "label": class index}: zero-padded waveforms with their padding mask,
    target [B, 1] (collate_tokens of one-token labels: no eos), prev_output_tokens [[eos]] per utterance, ntokens = B."""
    samples = [s for s in samples if s["source"] is not None]
    if len(samples) == 0:
        return {}
    source, padding_mask = _collate_audio([s["source"] for s in samples])
    B = len(samples)
    target = torch.tensor([[int(s["label"])] for s in samples], dtype=torch.long)
    return {"id": torch.LongTensor([s["id"] for s in samples]),
            "net_input": {"source": source, "padding_mask": padding_mask,
                          "prev_output_tokens": torch.full((B, 1), eos, dtype=torch.long), "task_name": "s2c"},
            "target": target, "target_lengths": torch.ones(B, dtype=torch.long), "task_name": "s2c", "ntokens": B}


def synthetic_sid_batch(B, n_samples, n_classes, seed=1, ragged=True, pin=False):
    """Speaker-identification batch through the s2c collater: waveforms N(0, 0.1^2) with lengths U{0.8 n .. n} (the
    first one n), speakers U{4 .. n_classes - 3} (the dictionary's specials and its trailing <mask> / <ctc_blank> are
    never a class)."""
    g = torch.Generator().manual_seed(seed)
    items = []
    for b in range(B):
        n = n_samples if (b == 0 or not ragged) else int(torch.randint(int(0.8 * n_samples), n_samples + 1, (1,), generator=g))
        items.append({"id": b, "source": torch.randn(n, generator=g) * 0.1,
                      "label": int(torch.randint(4, n_classes - 2, (1,), generator=g))})
    sample = collate_sid(items)
    return _pin(sample) if pin else sample


def collate_vc(samples, reduction_factor=2):
    """SpeechToSpeechDataset.collater (speecht5/data/speech_to_speech_dataset.py:169-228) over in-memory items
    {"id", "source": FloatTensor [N] waveform, "target": FloatTensor [L, odim] log-mel, "spkembs": FloatTensor [512],
    "audio_name", "tgt_name"}: zero-padded waveforms with their padding mask, the target frames padded, the decoder input
    = a zero frame then every r-th target frame ([r-1::r], last one dropped), stop labels 1 from the last real frame on,
    src_lengths / ntokens in waveform samples. Host-side work only."""
    samples = [s for s in samples if s["source"] is not None]
    if len(samples) == 0:
        return {}
    audio_sizes = [len(s["source"]) for s in samples]
    source, padding_mask = _collate_audio([s["source"] for s in samples])
    fbank_sizes = [len(s["target"]) for s in samples]
    fbanks = collate_frames([s["target"] for s in samples])
    sizes = torch.tensor(fbank_sizes, dtype=torch.long)
    r = reduction_factor
    if r > 1:
        fb_in, sizes_in = fbanks[:, r - 1::r], torch.div(sizes, r, rounding_mode="floor")
    else:
        fb_in, sizes_in = fbanks, sizes
    prev = torch.cat([fb_in.new_zeros((fb_in.shape[0], 1, fb_in.shape[2])), fb_in[:, :-1]], dim=1)
    labels = fbanks.new_zeros(fbanks.size(0), fbanks.size(1))
    for i, n in enumerate(fbank_sizes):
        labels[i, n - 1:] = 1.0
    spkembs = collate_frames([s["spkembs"] for s in samples], is_audio_input=True)
    net_input = {"source": source, "padding_mask": padding_mask, "prev_output_tokens": prev, "tgt_lengths": sizes_in,
                 "spkembs": spkembs, "task_name": "s2s"}
    return {"id": torch.LongTensor([s["id"] for s in samples]), "name": [s.get("audio_name") for s in samples],
            "tgt_name": [s.get("tgt_name") for s in samples], "net_input": net_input, "labels": labels,
            "dec_target": fbanks, "dec_target_lengths": sizes, "src_lengths": torch.LongTensor(audio_sizes),
            "task_name": "s2s", "ntokens": sum(audio_sizes), "target": fbanks}


def synthetic_vc_batch(B, n_samples, T_mel, seed=1, ragged=True, pin=False, odim=80, reduction_factor=2):
    """Voice-conversion batch through the s2s collater: source waveforms N(0, 0.1^2) with lengths U{0.8 n .. n},
    target log-mels N(0, 1) [L, odim] with L U{0.8 T .. T} (the first utterance n samples / T frames), 512-d
    x-vectors."""
    g = torch.Generator().manual_seed(seed)
    items = []
    for b in range(B):
        n, L = n_samples, T_mel
        if ragged and b > 0:
            n = int(torch.randint(int(0.8 * n_samples), n_samples + 1, (1,), generator=g))
            L = int(torch.randint(int(0.8 * T_mel), T_mel + 1, (1,), generator=g))
        items.append({"id": b, "source": torch.randn(n, generator=g) * 0.1,
                      "target": torch.randn(L, odim, generator=g), "spkembs": torch.randn(512, generator=g)})
    sample = collate_vc(items, reduction_factor)
    return _pin(sample) if pin else sample


def _span_lengths(rng, kind, count, length, other):
    """Span lengths of one row; each non-static kind consumes `count` draws from the stream, like the reference."""
    if kind == "static":
        return [length] * count
    if kind == "uniform":
        return list(rng.randint(other, length * 2 + 1, size=count))
    if kind == "normal":
        return [max(1, int(round(v))) for v in rng.normal(length, other, size=count)]
    if kind == "poisson":
        return [int(round(v)) for v in rng.poisson(length, size=count)]
    raise Exception("unknown mask selection " + kind)


def compute_mask_indices(shape, padding_mask, mask_prob, mask_length, mask_type="static", mask_other=0.0, min_masks=0,
                         no_overlap=False, min_space=0):
    """Span masks for the speech prenet: the host-side sampler behind `apply_hubert_mask`
    (speech_encoder_prenet.py:236-262), which in the reference is fairseq's `compute_mask_indices`
    (fairseq/data/data_utils.py:393-517, MIT licence, (c) Facebook). ATTRIBUTION: this is a re-statement of that
    routine, not an independent design -- a run seeded like the reference must mask the same frames, so the sequence of
    draws from the GLOBAL np.random stream has to be the reference's: one rand() for the batch-level span count, per
    row one more rand() when a padding mask is given, then that row's span lengths, then its span starts (choice
    without replacement); after all rows, one thinning choice() per row that has more masked frames than the shortest
    row. tests/test_ref_pin_cpu.py::test_host_mask_sampler_reproduces_the_reference_draws pins it bit for bit against
    the reference function. Returns a bool ndarray [B, T]. `no_overlap` (off in every SpeechT5 recipe) is not built."""
    import numpy as np
    if no_overlap:
        raise NotImplementedError("no_overlap span placement is not built (unused by the SpeechT5 recipes)")
    rng = np.random  # the global stream, on purpose
    rows, width = shape

    def span_count(n_valid):
        return max(min_masks, int(mask_prob * n_valid / float(mask_length) + rng.rand()))
    batch_count = span_count(width)
    per_row = []
    for r in range(rows):
        if padding_mask is None:
            n_valid, count = width, batch_count
        else:
            n_valid = width - int(padding_mask[r].long().sum().item())
            count = span_count(n_valid)
        spans = _span_lengths(rng, mask_type, count, mask_length, mask_other)
        if sum(spans) == 0:
            spans[0] = min(mask_length, n_valid - 1)
        shortest = min(spans)
        if n_valid - shortest <= count:
            shortest = n_valid - count - 1
        starts = rng.choice(n_valid - shortest, count, replace=False)
        covered = np.concatenate([np.arange(b, b + n) for b, n in zip(starts, spans)]) if count else np.zeros(0, int)
        per_row.append(np.unique(covered[covered < n_valid]))
    common = min(len(c) for c in per_row)
    out = np.zeros((rows, width), dtype=bool)
    for r, covered in enumerate(per_row):
        if len(covered) > common:
            covered = rng.choice(covered, common, replace=False)
        out[r, covered] = True
    return out


def draw_hubert_masks(prenet, batch_size, n_frames, frame_padding_mask):
    """Both mask draws of `apply_hubert_mask` (speech_encoder_prenet.py:234-272) for one batch, on the host, in the
    reference's order (time mask first, channel mask second). Returns (mask_indices [B,T] or None,
    mask_channel_indices [B,C] or None) as bool tensors; used by the trainer before a CUDA-graph replay."""
    mi = mc = None
    if prenet.mask_prob > 0:
        mi = torch.from_numpy(compute_mask_indices(
            (batch_size, n_frames), frame_padding_mask, prenet.mask_prob, prenet.mask_length, prenet.mask_selection,
            prenet.mask_other, min_masks=2, no_overlap=prenet.no_mask_overlap, min_space=prenet.mask_min_space))
    if getattr(prenet, "mask_channel_prob", 0.0) > 0:
        mc = torch.from_numpy(compute_mask_indices(
            (batch_size, prenet.embed_dim), None, prenet.mask_channel_prob, prenet.mask_channel_length,
            prenet.mask_channel_selection, prenet.mask_channel_other, no_overlap=prenet.no_mask_channel_overlap,
            min_space=prenet.mask_channel_min_space))
    return mi, mc


def _pin(obj):
    if torch.is_tensor(obj):
        return obj.pin_memory()
    if isinstance(obj, dict):
        return {k: _pin(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_pin(v) for v in obj)
    return obj

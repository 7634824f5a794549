"""CPU restatement of the speaker-identification head and its criterion, in float64 torch, from the reference's
definitions: SpeakerDecoderPostnet.forward (speecht5/models/modules/speaker_decoder_postnet.py:176-197) with
AngularMargin / AdditiveAngularMargin (:48-126), and label_smoothed_nll_loss + compute_accuracy of SpeechtoTextLoss
(speecht5/criterions/speech_to_text_loss.py:93-110, 340-372). Parameters are looked up by the reference's names."""
import math

import torch


def _bn(x, state, prefix, training, eps=1e-5):
    if training:
        mu, var = x.mean(0), x.var(0, unbiased=False)
    else:
        mu, var = state[prefix + "running_mean"].double(), state[prefix + "running_var"].double()
    return (x - mu) / torch.sqrt(var + eps) * state[prefix + "weight"].double() + state[prefix + "bias"].double()


def margin(cos, target, kind, m, s, easy_margin=False):
    """cos [B, N]; target [B] class indices (the one-hot rows of the reference)."""
    onehot = torch.nn.functional.one_hot(target, cos.shape[1]).double()
    if kind == "amsoftmax":
        return s * (cos - m * onehot)
    sine = torch.sqrt((1.0 - cos ** 2).clamp(0, 1))
    phi = cos * math.cos(m) - sine * math.sin(m)
    if easy_margin:
        phi = torch.where(cos > 0, phi, cos)
    else:
        phi = torch.where(cos > math.cos(math.pi - m), phi, cos - math.sin(math.pi - m) * m)
    return s * (onehot * phi + (1.0 - onehot) * cos)


def speaker_head(state, x, *, softmax_type="softmax", pooling_bn=True, embed_postnet=True, normalize=False,
                 scale=1.0, margin_m=0.0, easy_margin=False, target=None, training=True, prefix="speaker_decoder_postnet."):
    """Returns (logits, embed) like SpeakerDecoderPostnet.forward; `target` (class indices) gets the margin in training."""
    w = lambda k: state[prefix + k].double()  # noqa: E731
    x = x.double()
    if pooling_bn:
        x = _bn(x, state, prefix + "bn_pooling.", training)
    embed = _bn(x @ w("output_embedding.weight").t(), state, prefix + "bn_embedding.", training) if embed_postnet else x
    if softmax_type != "softmax" or normalize:
        xn = embed / embed.norm(dim=1, keepdim=True).clamp_min(1e-12)
        wt = w("output_projection.weight")
        wn = wt / wt.norm(dim=1, keepdim=True).clamp_min(1e-12)
        out = xn @ wn.t()
        if training and target is not None and softmax_type != "softmax":
            out = margin(out, target, softmax_type, margin_m, scale, easy_margin)
    else:
        out = embed @ w("output_projection.weight").t()
    return out, embed


def label_smoothed_ce(logits, target, eps, ignore_index=1):
    """(loss, nll, n_correct, total) summed over rows, as SpeechtoTextLoss.compute_loss / compute_accuracy give them."""
    lprobs = torch.log_softmax(logits.double(), dim=-1)
    t = target.reshape(-1)
    keep = t.ne(ignore_index)
    nll = -lprobs.gather(1, t[:, None].clamp_min(0))[:, 0] * keep
    smooth = -lprobs.sum(-1) * keep
    eps_i = eps / (lprobs.size(-1) - 1)
    loss = ((1.0 - eps - eps_i) * nll + eps_i * smooth).sum()
    correct = (lprobs.argmax(1).eq(t) & keep).sum()
    return loss, nll.sum(), int(correct), int(keep.sum())

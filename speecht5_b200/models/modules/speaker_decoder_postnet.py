"""Speaker-identification head (speecht5/models/modules/speaker_decoder_postnet.py:129-197) on the H100 kernels: the
pooled decoder (or encoder) state -> optional BatchNorm -> optional embedding projection + BatchNorm -> class logits,
either a plain projection or cosines of L2-normalised embedding and class weight rows with an additive (AM) or
angular (AAM) margin on the target class in training. Same parameter names as the reference, so its checkpoints load."""
import torch
import torch.nn as nn

from ... import ops
from ..._lib import MARGIN_AAM, MARGIN_AM


class SpeakerDecoderPostnet(nn.Module):
    def __init__(self, embed_dim, class_num, args):
        super().__init__()
        self.embed_dim = embed_dim
        self.class_num = class_num
        self.no_pooling_bn = getattr(args, "sid_no_pooling_bn", False)
        self.no_embed_postnet = getattr(args, "sid_no_embed_postnet", False)
        self.normalize_postnet = getattr(args, "sid_normalize_postnet", False)
        self.softmax_head = getattr(args, "sid_softmax_type", "softmax")
        d = getattr(args, "decoder_output_dim", args.decoder_embed_dim)
        self.bn_pooling = None if self.no_pooling_bn else nn.BatchNorm1d(d)
        if not self.no_embed_postnet:
            self.output_embedding = nn.Linear(d, embed_dim, bias=False)
            self.bn_embedding = nn.BatchNorm1d(embed_dim)
        else:
            self.output_embedding = self.bn_embedding = None
            self.embed_dim = d
        self.output_projection = nn.Linear(self.embed_dim, class_num, bias=False)
        # (mode, scale, margin, easy_margin) of the margin layer (:166-171); None: plain softmax head
        self.margin = None
        if self.softmax_head == "amsoftmax":
            self.margin = (MARGIN_AM, float(args.softmax_scale), float(args.softmax_margin), 0)
        elif self.softmax_head == "aamsoftmax":
            self.margin = (MARGIN_AAM, float(args.softmax_scale), float(args.softmax_margin),
                           int(bool(args.softmax_easy_margin)))
        if self.output_embedding is not None:  # (:172-174)
            nn.init.normal_(self.output_embedding.weight, mean=0, std=embed_dim ** -0.5)
        nn.init.normal_(self.output_projection.weight, mean=0, std=class_num ** -0.5)

    def forward(self, x, target=None):
        """x [B, C]; target: class indices [B] (the reference takes their one-hot rows), the column that receives the
        margin in training. Returns (logits [B, class_num] fp32, embedding [B, embed_dim])."""
        if self.bn_pooling is not None:
            x = ops.batch_norm_act(x, self.bn_pooling, self.training)
        if self.output_embedding is not None:
            embed = ops.batch_norm_act(ops.linear(x, self.output_embedding.weight), self.bn_embedding, self.training)
        else:
            embed = x
        if self.margin is not None or self.normalize_postnet:
            w = self.output_projection.weight
            output = ops.cosine(ops.l2_normalize_rows(embed), ops.l2_normalize_rows(w, grad_key=("lin", id(w))))
            if self.training and target is not None and self.margin is not None:
                output = ops.margin_logits(output, target, self.margin)
        else:
            output = ops.linear(embed, self.output_projection.weight, (), out_dtype=torch.float32)
        return output, embed


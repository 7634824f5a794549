"""Pre-training extras on the device (SURVEY section 8a row 22): the HuBERT-style masked-prediction head
(speecht5/models/modules/speech_encoder_postnet.py:26-124), the Gumbel vector quantizer
(fairseq/modules/gumbel_vector_quantizer.py:13-202 in the SpeechT5 configuration: 100 variables x 2 groups, one linear
projection, time-first input) and the code mixing of models/speecht5.py:858-872.

Used by the speech pre-training branch of T5TransformerModel.forward (target_list / --use-codebook); the criteria
are criterions/speech_pretrain_criterion.py and text_pretrain_criterion.py. The two projections run on the wgmma GEMM
(ops.linear); the rest acts on [frames, classes]-sized tensors (cosine similarities against the label embeddings,
Gumbel-softmax over 100 variables, a 200 x d codebook product) and is issued as torch calls. Checked on the CPU against
oracle/pretrain_oracle.py through the kernel emulation (tests/test_frontend_cpu.py), forward and backward.

As in the oracle, the random draws of the reference (Gumbel noise inside F.gumbel_softmax, torch.randperm of the time
steps) can be passed in explicitly so that a run can be compared draw for draw."""
import torch
import torch.nn as nn

from . import ops


class SpeechEncoderPostnet(nn.Module):
    """Parameter names of the reference: `label_embs_concat`, `final_proj.{weight,bias}` (target GLU off, as in every
    SpeechT5 recipe)."""

    def __init__(self, num_classes, encoder_embed_dim=768, final_dim=256, logit_temp=0.1, untie_final_proj=True,
                 skip_masked=False, skip_nomask=False, target_glu=False):
        super().__init__()
        if target_glu:
            raise NotImplementedError("target_glu is not built (False in every SpeechT5 recipe)")
        self.num_classes = list(num_classes)
        self.logit_temp, self.untie_final_proj = logit_temp, untie_final_proj
        self.skip_masked, self.skip_nomask = skip_masked, skip_nomask
        self.label_embs_concat = nn.Parameter(torch.empty(sum(self.num_classes), final_dim).uniform_())
        self.final_proj = nn.Linear(encoder_embed_dim, final_dim * (len(self.num_classes) if untie_final_proj else 1))

    def compute_nce(self, x, pos, negs):  # :61-74
        neg_is_pos = (pos == negs).all(-1)
        targets = torch.cat([pos.unsqueeze(0), negs], dim=0)
        logits = torch.cosine_similarity(x.float(), targets.float(), dim=-1).type_as(x) / self.logit_temp
        if neg_is_pos.any():
            logits[1:][neg_is_pos] = float("-inf")
        return logits.transpose(0, 1)

    def forward(self, x, padding_mask, mask_indices, target_list):
        """x [B, T, d] encoder output; returns {"logit_m_list", "logit_u_list", "padding_mask"} (:76-124)."""
        label_embs_list = self.label_embs_concat.split(self.num_classes, 0)

        def head(sel):
            frames = x[sel]  # [n, d] gather of the selected frames
            if frames.shape[0] == 0:
                proj = frames.new_zeros((0, self.final_proj.out_features))
            else:
                proj = ops.linear(frames.unsqueeze(0), self.final_proj.weight, self.final_proj.bias)[0]
            chunks = proj.chunk(len(target_list), dim=-1) if self.untie_final_proj else [proj] * len(target_list)
            out = []
            for i, (px, t) in enumerate(zip(chunks, target_list)):
                y = torch.index_select(label_embs_list[i], 0, t[sel].long())
                negs = label_embs_list[i].unsqueeze(1).expand(-1, px.size(0), -1)
                out.append(self.compute_nce(px, y, negs))
            return out

        m = None if self.skip_masked else head(torch.logical_and(~padding_mask, mask_indices))
        u = None if self.skip_nomask else head(torch.logical_and(~padding_mask, ~mask_indices))
        return {"logit_m_list": m if m is not None else [None for _ in target_list],
                "logit_u_list": u if u is not None else [None for _ in target_list], "padding_mask": padding_mask}


class GumbelVectorQuantizer(nn.Module):
    """Parameter names of the reference: `vars` [1, groups*num_vars, vq_dim/groups], `weight_proj.{weight,bias}`."""

    def __init__(self, dim=768, num_vars=100, temp=(2.0, 0.5, 0.999995), groups=2, vq_dim=768):
        super().__init__()
        assert vq_dim % groups == 0
        self.groups, self.num_vars, self.input_dim = groups, num_vars, dim
        self.vars = nn.Parameter(torch.empty(1, groups * num_vars, vq_dim // groups).uniform_())
        self.weight_proj = nn.Linear(dim, groups * num_vars)
        nn.init.normal_(self.weight_proj.weight, mean=0, std=1)
        nn.init.zeros_(self.weight_proj.bias)
        self.max_temp, self.min_temp, self.temp_decay = temp
        self.curr_temp = self.max_temp

    def set_num_updates(self, num_updates):
        self.curr_temp = max(self.max_temp * self.temp_decay ** num_updates, self.min_temp)

    def forward(self, x, gumbel_noise=None):
        result = {"num_vars": self.num_vars * self.groups}
        bsz, tsz, fsz = x.shape
        logits = ops.linear(x, self.weight_proj.weight, self.weight_proj.bias, out_dtype=torch.float32)
        logits = logits.reshape(bsz * tsz * self.groups, -1)
        k = logits.argmax(-1)
        hard_x = torch.zeros_like(logits).scatter_(-1, k.view(-1, 1), 1.0).view(bsz * tsz, self.groups, -1)
        hard_probs = hard_x.float().mean(dim=0)
        result["code_perplexity"] = torch.exp(-torch.sum(hard_probs * torch.log(hard_probs + 1e-7), dim=-1)).sum()
        avg_probs = torch.softmax(logits.view(bsz * tsz, self.groups, -1).float(), dim=-1).mean(dim=0)
        result["prob_perplexity"] = torch.exp(-torch.sum(avg_probs * torch.log(avg_probs + 1e-7), dim=-1)).sum()
        result["temp"] = self.curr_temp
        if self.training:
            if gumbel_noise is None:
                gumbel_noise = -torch.empty_like(logits, dtype=torch.float).exponential_().log()
            y_soft = ((logits.float() + gumbel_noise) / self.curr_temp).softmax(-1)
            idx = y_soft.argmax(-1, keepdim=True)
            y_hard = torch.zeros_like(y_soft).scatter_(-1, idx, 1.0)
            sel = y_hard - y_soft.detach() + y_soft  # straight-through estimator of F.gumbel_softmax(hard=True)
        else:
            sel = hard_x
        sel = sel.view(bsz * tsz, -1)
        q = (sel.unsqueeze(-1) * self.vars.float()).view(bsz * tsz, self.groups, self.num_vars, -1).sum(-2)
        result["x"] = q.view(bsz, tsz, -1).to(x.dtype)
        return result


def mix_codes(encoder_out_btc, q_x, codebook_prob, perm=None):
    """models/speecht5.py:866-872: a random `codebook_prob` fraction of the TIME steps, shared by the whole batch, is
    replaced by the quantized vectors. perm = the torch.randperm(T) draw (sampled here when not given)."""
    T = q_x.size(1)
    if perm is None:
        perm = torch.randperm(T, device=q_x.device)
    w = q_x.new_zeros(T)
    w[perm[: int(T * codebook_prob)]] = 1.0
    return w.view(-1, 1) * q_x + (1.0 - w).view(-1, 1) * encoder_out_btc

"""CPU ORACLE (test infrastructure, NOT product code): the voice-conversion (s2s) composition of microsoft/SpeechT5 from
the restated pieces -- the waveform prenet of oracle/speecht5_oracle_asr.py, the encoder / decoder stacks and the speech
decoder pre/post-nets of oracle/speecht5_oracle.py -- and the s2s form of the TTS criterion. Paths cited as file:line
under /root/reference/SpeechT5/speecht5. Pinned to the reference's own run by tests/golden/ref_vc_tiny.npz
(tests/golden/make_golden_vc.py, tests/test_vc_cpu.py)."""
import torch
import torch.nn as nn

from .speecht5_oracle import (SpeechDecoderPostnet, SpeechDecoderPrenet, TransformerDecoder, TransformerEncoder,
                              init_bert_params, tts_loss)
from .speecht5_oracle_asr import SpeechEncoderPrenet


class T5TransformerModelVCOracle(nn.Module):
    """models/speecht5.py:47-116 + the s2s branch of forward (:786-963): speech prenet -> encoder -> speech decoder prenet
    with the x-vector merged in ("pre", :899-902) -> decoder (cross-attention of every layer returned, :921-923) ->
    speech decoder post-net. Returns (before, after, stop logits, [attn per layer])."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        self.encoder = TransformerEncoder(args)
        self.decoder = TransformerDecoder(args)
        self.speech_encoder_prenet = SpeechEncoderPrenet(args)
        self.speech_decoder_prenet = SpeechDecoderPrenet(args.speech_odim, args)
        self.speech_decoder_postnet = SpeechDecoderPostnet(args.speech_odim, args)
        self.reduction_factor = args.reduction_factor
        if args.bert_init:
            self.apply(init_bert_params)

    def encode(self, source, padding_mask):
        x, enc_pad, _ = self.speech_encoder_prenet(source, padding_mask, None, None)
        return self.encoder(x, enc_pad)

    def forward(self, source=None, padding_mask=None, prev_output_tokens=None, tgt_lengths=None, spkembs=None, **unused):
        encoder_output = self.encode(source, padding_mask)
        dec_in, tgt_mask = self.speech_decoder_prenet(prev_output_tokens, tgt_lengths, spkembs)
        decoder_output, extra = self.decoder(dec_in, tgt_mask, encoder_output, alignment_layer=-1)
        return self.speech_decoder_postnet(decoder_output) + (extra["attn"][0],)

    @torch.no_grad()
    def generate_speech(self, source, padding_mask, spkembs=None, **kwargs):
        """models/speecht5.py:1188-1249, speech input: the "threshold" key sets the threshold, minlenratio AND maxlenratio
        (defaults 0.5 / 0.0 / 10.0). The decoder is re-run on the prefix every step (equal to the reference's
        incremental state: causal self-attention, prenet dropout 0)."""
        assert source.size(0) == 1
        threshold = kwargs.get("threshold", 0.5)
        minlenratio = kwargs.get("threshold", 0.0)
        maxlenratio = kwargs.get("threshold", 10.0)
        encoder_out = self.encode(source, padding_mask)
        r, odim = self.reduction_factor, self.speech_decoder_postnet.odim
        T_enc = encoder_out["encoder_out"][0].size(0)
        maxlen, minlen = int(T_enc * maxlenratio / r), int(T_enc * minlenratio / r)
        ys = encoder_out["encoder_out"][0].new_zeros(1, 1, odim)
        outs, probs, attns, idx = [], [], [], 0
        while True:
            idx += 1
            decoder_in, _ = self.speech_decoder_prenet(ys, spkembs=spkembs)
            z, extra = self.decoder(decoder_in, None, encoder_out, alignment_layer=-1)
            outs.append(self.speech_decoder_postnet.feat_out(z[0, -1]).view(r, odim))
            probs.append(torch.sigmoid(self.speech_decoder_postnet.prob_out(z[0, -1])))
            ys = torch.cat((ys, outs[-1][-1].view(1, 1, odim)), dim=1)
            attns.append(torch.stack([a[0, :, -1:, :] for a in extra["attn"][0]], dim=0))
            if int((probs[-1] >= threshold).sum()) > 0 or idx >= maxlen:
                if idx < minlen:
                    continue
                mel = torch.cat(outs, dim=0).unsqueeze(0).transpose(1, 2)
                mel = mel + self.speech_decoder_postnet.postnet(mel)
                return mel.transpose(2, 1).squeeze(0), torch.cat(probs, dim=0), torch.cat(attns, dim=2)


def vc_loss(model, model_out, sample, **kw):
    """criterions/text_to_speech_loss.py:154-214 for an s2s batch: the guided-attention input lengths are the conv front
    end's frame counts of the waveform lengths (:198-206, SpeechEncoderPrenet.get_src_lengths)."""
    ilens = model.speech_encoder_prenet.feature_extractor.get_out_seq_lens_tensor(sample["src_lengths"])
    return tts_loss(model_out, dict(sample, src_lengths=ilens), reduction_factor=model.reduction_factor, **kw)

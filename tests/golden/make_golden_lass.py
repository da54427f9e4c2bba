#!/usr/bin/env python
"""Generate the sound-extraction fixtures (lass_small.npz, lass_shipped.npz) by running the REFERENCE's own
sound_extraction/model/LASSNet.py (Text_Encoder + UNetRes_FiLM) and sound_extraction/utils/stft.py STFT on CPU fp32,
the way SoundExtraction.inference (audio-chatgpt.py:689-710) calls them: STFT.transform on a [1, N] clip, the
transposed magnitude view into the model with ['[CLS] ' + text], mask * magnitude, STFT.inverse.

Run in the build container only (needs the reference tree, which does not travel to the GPU box):

    python tests/golden/make_golden_lass.py

Nothing reaches the network: HF_HUB_OFFLINE=1 is set first, and
- BertModel.from_pretrained builds BertModel(BertConfig(bert-mini shape of the spec config)) locally;
- BertTokenizer.from_pretrained returns a stub whose __call__ hands back the stored ids and attention mask;
- librosa (not installed here) is a stub with the three librosa.util functions stft.py uses: pad_center, tiny and
  normalize(norm=None), which returns its input.
Weights are specs.synth_lass(cfg, seed) and clips specs.synth_lass_wav(n, seed): the fixtures store seeds and outputs,
and the tests regenerate the inputs.

lass_small: n_fft 256 (F = 129, the smallest F the UNet's skips close on), hop 128, B = 2 clips of 11 557 samples
(T = 91, ragged), two captions of different lengths, LASS_SMALL (bert-mini with a 1000-token vocabulary): every output.
lass_shipped: the tool's shape (n_fft 1024, hop 512, one 10 s 32 kHz clip: T = 626, F = 513), LASS: cond, per-frame
sums of the mask and logits, a strided sample of both, and samples of the STFT buffers and the window sum.
"""
import os
import sys
import types
from unittest import mock

os.environ["HF_HUB_OFFLINE"] = "1"

import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, ROOT, save, specs  # noqa: E402

SEED_W, SEED_IDS, SEED_WAV = 6060, 61, 62
SMALL_N, SMALL_FFT, SHIP_N = 128 * 90 + 37, 256, 320000
SAMPLE_STRIDE = 97


def librosa_stub():
    lib = types.ModuleType("librosa")
    util = types.ModuleType("librosa.util")

    def pad_center(data, size, axis=-1, **kw):
        n = data.shape[axis]
        lpad = int((size - n) // 2)
        lengths = [(0, 0)] * data.ndim
        lengths[axis] = (lpad, int(size - n - lpad))
        return np.pad(data, lengths, **kw)

    util.pad_center = pad_center
    util.tiny = lambda x: np.finfo(np.asarray(x).dtype if np.asarray(x).dtype.kind == "f" else np.float32).tiny
    util.normalize = lambda S, norm=np.inf, **kw: S if norm is None else None
    lib.util = util
    return {"librosa": lib, "librosa.util": util}


class StubTokenizer:
    def __init__(self, ids, mask):
        self.ids, self.mask = ids, mask

    def __call__(self, caption, add_special_tokens=False, padding=True, return_tensors="pt"):
        assert not add_special_tokens and padding and len(caption) == self.ids.shape[0]
        return {"input_ids": self.ids.clone(), "attention_mask": self.mask.clone()}


def run(cfg, n_fft, wav, ids, mask):
    from transformers import BertConfig, BertModel, BertTokenizer
    bcfg = dict(vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"], num_hidden_layers=cfg["num_layers"],
                num_attention_heads=cfg["num_heads"], intermediate_size=cfg["intermediate_size"],
                max_position_embeddings=cfg["max_position_embeddings"], type_vocab_size=cfg["type_vocab_size"],
                layer_norm_eps=cfg["layer_norm_eps"])

    def local_bert(name, add_pooling_layer=True, **kw):
        assert name == "prajjwal1/bert-mini"
        return BertModel(BertConfig(**bcfg, **kw), add_pooling_layer=add_pooling_layer)

    with mock.patch.dict(sys.modules, librosa_stub()), \
            mock.patch.object(BertModel, "from_pretrained", staticmethod(local_bert)), \
            mock.patch.object(BertTokenizer, "from_pretrained", staticmethod(lambda name: StubTokenizer(ids, mask))):
        sys.path.insert(0, REF)
        from sound_extraction.model.LASSNet import LASSNet
        from sound_extraction.utils.stft import STFT, window_sumsquare
        stft = STFT(filter_length=n_fft, hop_length=n_fft // 2, win_length=n_fft)
        model = LASSNet("cpu")
        sd = specs.synth_lass(cfg, SEED_W)
        keys = list(model.state_dict().keys())
        assert keys == list(specs.lass_param_shapes(cfg)), "lass_param_shapes differs from the reference key order"
        model.load_state_dict(sd, strict=True)
        model.eval()
        with torch.no_grad():
            mag, phase = stft.transform(wav)
            x = mag.transpose(2, 1).unsqueeze(1)                  # [B, 1, T, F], the tool's transposed view
            captions = ["[CLS] query"] * ids.shape[0]
            m = model(x, captions)
            cond = model.text_embedder(ids, mask)[0]
            logits = model.UNet(x, cond, cond)
            est = (m * x).squeeze(1).permute(0, 2, 1)
            out = stft.inverse(est, phase)
        ws = window_sumsquare("hann", mag.shape[-1], hop_length=n_fft // 2, win_length=n_fft, n_fft=n_fft, dtype=np.float32)
        return dict(stft=stft, mag=mag, phase=phase, mask=m, cond=cond, logits=logits, out=out, ws=ws, keys=keys)


def main():
    torch.set_grad_enabled(False)
    ids, mask = specs.synth_lass_ids(specs.LASS_SMALL, [9, 5], SEED_IDS)
    wav = torch.stack([specs.synth_lass_wav(SMALL_N, SEED_WAV), specs.synth_lass_wav(SMALL_N, SEED_WAV + 1)])
    r = run(specs.LASS_SMALL, SMALL_FFT, wav, ids, mask)
    save("lass_small", seed_w=SEED_W, seed_wav=SEED_WAV, n=SMALL_N, n_fft=SMALL_FFT, ids=ids, mask=mask, mag=r["mag"],
         phase=r["phase"], mask_out=r["mask"], logits=r["logits"], cond=r["cond"], wav_out=r["out"],
         ws=r["ws"], keys=np.array(r["keys"]))

    ids1, mask1 = specs.synth_lass_ids(specs.LASS, [11], SEED_IDS + 1)
    wav1 = specs.synth_lass_wav(SHIP_N, SEED_WAV + 2)[None]
    r = run(specs.LASS, specs.LASS_FFT, wav1, ids1, mask1)
    fb, ib = r["stft"].forward_basis, r["stft"].inverse_basis
    s = SAMPLE_STRIDE
    save("lass_shipped", seed_w=SEED_W, seed_wav=SEED_WAV + 2, n=SHIP_N, ids=ids1, mask=mask1, cond=r["cond"],
         mask_rows=r["mask"].double().sum(-1).reshape(-1), logits_rows=r["logits"].double().sum(-1).reshape(-1),
         mask_sample=r["mask"].reshape(-1)[::s], logits_sample=r["logits"].reshape(-1)[::s],
         mag_sample=r["mag"].reshape(-1)[::s], wav_out_sample=r["out"].reshape(-1)[::s],
         wav_out_sum=np.array([r["out"].double().sum().item(), r["out"].double().abs().sum().item()]),
         fwd_sample=fb.reshape(-1)[::s], inv_sample=ib.reshape(-1)[::s],
         fwd_sum=np.array([fb.double().sum().item(), fb.double().abs().sum().item()]),
         inv_sum=np.array([ib.double().sum().item(), ib.double().abs().sum().item()]),
         ws_sample=r["ws"][::s], ws_sum=np.array([r["ws"].astype(np.float64).sum()]), sample_stride=s)


if __name__ == "__main__":
    main()

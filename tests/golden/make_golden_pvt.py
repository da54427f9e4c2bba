#!/usr/bin/env python
"""Generate the sound-event-detection fixtures (pvt_small.npz, pvt_shipped.npz) by running the REFERENCE's own PVT
(audio_detection/audio_infer/pytorch/models.py) on CPU fp32 in eval mode, the way the SoundDetection tool calls it
(audio-chatgpt.py:612-673): ``model(waveform, None)``.

Run in the build container only (needs the reference tree, which does not travel to the GPU box):

    python tests/golden/make_golden_pvt.py

The reference module imports packages that are not installed here, only for names its eval forward never needs, so
they are stubbed in sys.modules: timm.models.layers (DropPath as an identity module, to_2tuple, trunc_normal_ =
torch's), timm.models.helpers, mmcv.runner, mmdet.utils, torchlibrosa.augmentation (empty shells holding the imported
names) and torchlibrosa.stft (make_golden_clap_score's restatement of torchlibrosa 0.1.0).

- pvt_shipped: ``PVT(32000, 1024, 320, 64, 50, 14000, 527)`` as the tool builds it, on one 10 s clip.
- pvt_small: the reference's ``PVT.forward`` on a module assembled from the reference's own parts at the
  specs.PVT_SMALL sizes (the sizes of PyramidVisionTransformerV2 are fixed inside ``PVT.__init__``), on two clips: one
  whose stage grids leave a remainder in every sr gather and one whose grids divide evenly.
Weights are specs.synth_pvt(cfg, seed), loaded strictly; clips are specs.synth_pvt_wav(n, seed).  Neither is stored: the
fixtures keep the seeds, per-clip sums, the reference's state-dict keys and shapes, and outputs only.
"""
import os
import sys
import types
from functools import partial

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, ROOT, save, specs, stats  # noqa: E402
from make_golden_clap_score import torchlibrosa_shim  # noqa: E402

SEED_SMALL, SEED_SHIPPED = 3030, 3031
CLIP_SEED = 33
SMALL_LENS = (8250, 5040)     # stage grids 26/13/7/4 rows (a remainder for sr 8, 4 and 2) and 16/8/4/2 rows (none)
SHIPPED_LEN = 320000          # 10 s at 32 kHz: 1001 frames
ROW_STEP = 37                 # framewise rows kept in pvt_shipped (coprime to the 32-fold repeat)


def import_reference_models():
    def shell(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules.setdefault(name, m)
        return sys.modules[name]

    class DropPath(nn.Module):
        def __init__(self, drop_prob=None):
            super().__init__()
            self.drop_prob = drop_prob

        def forward(self, x):
            assert not self.training
            return x

    class SpecAugmentation(nn.Module):
        def __init__(self, **kw):
            super().__init__()

        def forward(self, x):
            assert not self.training
            return x

    unused = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("stub"))   # noqa: E731
    shell("timm"); shell("timm.models")
    shell("timm.models.layers", DropPath=DropPath, to_2tuple=lambda v: v if isinstance(v, tuple) else (v, v),
          trunc_normal_=nn.init.trunc_normal_)
    shell("timm.models.helpers", load_pretrained=unused)
    shell("mmdet"); shell("mmdet.utils", get_root_logger=unused)
    shell("mmcv", runner=shell("mmcv.runner", load_checkpoint=unused, _load_checkpoint=unused, load_state_dict=unused))
    shell("torchlibrosa")
    sys.modules.setdefault("torchlibrosa.stft", torchlibrosa_shim())
    shell("torchlibrosa.augmentation", SpecAugmentation=SpecAugmentation)
    sys.path.insert(0, os.path.join(REF, "audio_detection"))
    import audio_infer.pytorch.models as models
    return models


def small_reference(models, cfg):
    """The reference's PVT with PVT.__init__'s attributes built at cfg's sizes from the reference's own classes."""
    m = models.PVT.__new__(models.PVT)
    nn.Module.__init__(m)
    m.spectrogram_extractor = models.Spectrogram(n_fft=cfg["window_size"], hop_length=cfg["hop_size"], win_length=cfg["window_size"],
                                                 window="hann", center=True, pad_mode="reflect", freeze_parameters=True)
    m.logmel_extractor = models.LogmelFilterBank(sr=cfg["sample_rate"], n_fft=cfg["window_size"], n_mels=cfg["mel_bins"],
                                                 fmin=cfg["fmin"], fmax=cfg["fmax"], ref=1.0, amin=1e-10, top_db=None,
                                                 freeze_parameters=True)
    m.time_shift = models.TimeShift(0, 10)
    m.spec_augmenter = models.SpecAugmentation(time_drop_width=64, time_stripes_num=2, freq_drop_width=8, freq_stripes_num=2)
    m.bn0 = nn.BatchNorm2d(64)
    m.pvt_transformer = models.PyramidVisionTransformerV2(
        tdim=1001, fdim=64, patch_size=7, stride=4, in_chans=1, num_classes=cfg["classes_num"], embed_dims=list(cfg["embed_dims"]),
        depths=list(cfg["depths"]), num_heads=list(cfg["num_heads"]), mlp_ratios=list(cfg["mlp_ratios"]), qkv_bias=True,
        qk_scale=None, drop_rate=0.0, drop_path_rate=0.1, sr_ratios=list(cfg["sr_ratios"]),
        norm_layer=partial(nn.LayerNorm, eps=1e-6), num_stages=4)
    m.avgpool = nn.AdaptiveAvgPool1d(1)
    m.fc_audioset = nn.Linear(cfg["embed_dims"][-1], cfg["classes_num"], bias=True)
    return m


def run(model, wav):
    """model(wav, None) with the pre-sigmoid logits and the four stage outputs ([B, N_i, C_i] after norm{i}) captured."""
    cap = {}
    hooks = [model.fc_audioset.register_forward_hook(lambda mod, i, o: cap.__setitem__("logits", o.detach().clone()))]
    for i in range(4):
        hooks.append(getattr(model.pvt_transformer, f"norm{i + 1}").register_forward_hook(
            lambda mod, inp, o, i=i: cap.__setitem__(f"stage{i + 1}", o.detach().clone())))
    with torch.no_grad():
        out = model(wav, None)
    for h in hooks:
        h.remove()
    return out, cap


def keys_and_shapes(model):
    sd = model.state_dict()
    return dict(ref_keys=np.array(list(sd.keys())), ref_shapes=np.array([",".join(str(v) for v in t.shape) for t in sd.values()]))


def main():
    models = import_reference_models()

    cfg = specs.PVT_SMALL
    model = small_reference(models, cfg).eval()
    model.load_state_dict(specs.synth_pvt(cfg, SEED_SMALL), strict=True)
    arrs = dict(weight_seed=np.array(SEED_SMALL), clip_seed=np.array(CLIP_SEED), clip_lens=np.array(SMALL_LENS), **keys_and_shapes(model))
    for k, n in enumerate(SMALL_LENS):
        wav = specs.synth_pvt_wav(n, CLIP_SEED + k)
        out, cap = run(model, wav[None])
        assert list(cap["stage1"].shape[1:]) == [np.prod(specs.pvt_grids(cfg, n)[0]), cfg["embed_dims"][0]]
        print(f"small clip {n}: grids {specs.pvt_grids(cfg, n)}, logits rms {cap['logits'].pow(2).mean().sqrt():.3f}, "
              f"clipwise in [{out['clipwise_output'].min():.3f}, {out['clipwise_output'].max():.3f}]")
        arrs.update({f"clip_stats{k}": stats(wav), f"framewise{k}": out["framewise_output"], f"clipwise{k}": out["clipwise_output"],
                     f"logits{k}": cap["logits"]})
        if k == 0:
            arrs.update({f"stage{i + 1}": cap[f"stage{i + 1}"] for i in range(4)})
    save("pvt_small", **arrs)

    cfg = specs.PVT_SHIPPED
    model = models.PVT(sample_rate=32000, window_size=1024, hop_size=320, mel_bins=64, fmin=50, fmax=14000, classes_num=527).eval()
    model.load_state_dict(specs.synth_pvt(cfg, SEED_SHIPPED), strict=True)
    wav = specs.synth_pvt_wav(SHIPPED_LEN, CLIP_SEED)
    out, cap = run(model, wav[None])
    frame = out["framewise_output"]
    top = np.argsort(np.max(frame[0].numpy(), axis=0))[::-1][:10]
    print(f"shipped: framewise {tuple(frame.shape)}, logits rms {cap['logits'].pow(2).mean().sqrt():.3f}, top-10 {top.tolist()}")
    save("pvt_shipped", weight_seed=np.array(SEED_SHIPPED), clip_seed=np.array(CLIP_SEED), clip_len=np.array(SHIPPED_LEN),
         clip_stats=stats(wav), logits=cap["logits"], clipwise=out["clipwise_output"], framewise_rows=frame[:, ::ROW_STEP],
         row_step=np.array(ROW_STEP), framewise_shape=np.array(frame.shape), top10=top.copy(), **keys_and_shapes(model))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    torch.set_num_threads(os.cpu_count() or 1)
    main()

"""Drop-in for ``wav_evaluation.models.CLAPWrapper``: the CLAP model with which the text-to-audio tool scores its
candidate clips against the prompt and keeps the best one (T2A.select_best_audio, audio-chatgpt.py:185-199).

Reference: text_to_audio/Make_An_Audio/wav_evaluation/models/CLAPWrapper.py, clap.py and audio.py (Cnn14 on
torchlibrosa features, BERT text tower, CLAP Projections).  Same constructor ``(model_fp, config_path,
use_cuda=False)``, same ``args``, ``tokenizer``, ``token_keys``, ``config_as_str``, ``model_fp``, ``use_cuda`` and
``file_path`` attributes, same ``get_text_embeddings``, ``get_audio_embeddings(audio_files, resample)`` (paths or
``(tensor, sample_rate)`` tuples), ``compute_similarity`` and ``cal_clap_score``.  Audio decoding (torchaudio.load)
and tokenization stay on the host; everything else runs in libagpt_b200.so (csrc/clap_score.cu, csrc/clap.cu).  CUDA
only, inference only.

Differences from the reference:
- it imports on torch 2.x (the reference imports ``torch._six``, which no longer exists);
- ``use_cuda=False`` or a machine without CUDA raises: there is no CPU fallback;
- the engines are cached for one checkpoint, keyed by (realpath, size, mtime_ns) of ``model_fp`` and the config
  text: the tool builds a new CLAPWrapper per request, which would otherwise re-read and re-pack about 190 M
  parameters every time;
- the text tower's architecture comes from ``AutoConfig.from_pretrained(text_model)`` (head count, LayerNorm eps)
  and the checkpoint's shapes, instead of ``AutoModel.from_pretrained``, whose weights the checkpoint overwrites;
- checkpoint keys the scorer never uses are accepted and ignored: ``fc_audioset.*``, ``num_batches_tracked``, BERT's
  ``pooler.*`` and ``embeddings.position_ids``;
- audio must be mono (a 1-D clip or one channel): the reference would flatten the channels of a multi-channel
  file into one signal.
"""
from __future__ import annotations

import argparse
import ctypes as C
import math
import os
import random
import re

import numpy as np
import torch

from ... import _lib, specs

_CACHE = {}   # one entry: (realpath, size, mtime_ns, config text, device index) -> _Scorer


def read_config_as_args(config_path, args=None, is_config_str=False):
    """wav_evaluation/models/utils.py read_config_as_args: the YAML's top-level keys as an argparse.Namespace."""
    import yaml
    if is_config_str:
        yml = yaml.load(config_path, Loader=yaml.FullLoader)
    else:
        with open(config_path) as f:
            yml = yaml.load(f, Loader=yaml.FullLoader)
    if args is not None:
        for k, v in yml.items():
            if k in args.__dict__:
                args.__dict__[k] = v
        return args
    return argparse.Namespace(**yml)


def scorer_config(args, state_dict, bert_config):
    """The specs.CLAP_SCORER-style config of a checkpoint: the YAML values plus the BERT shape read from the weights and
    the head count / LayerNorm eps of the transformers BertConfig."""
    if getattr(bert_config, "hidden_act", "gelu") != "gelu":
        raise NotImplementedError(f"audiogpt_b200.CLAPWrapper: hidden_act={bert_config.hidden_act!r} (only 'gelu')")
    b = "caption_encoder.base."
    word = state_dict[b + "embeddings.word_embeddings.weight"]
    H = int(word.shape[1])
    n_layers = len({k.split(".")[4] for k in state_dict if k.startswith(b + "encoder.layer.")})
    bert = dict(vocab_size=int(word.shape[0]), hidden_size=H,
                max_position_embeddings=int(state_dict[b + "embeddings.position_embeddings.weight"].shape[0]),
                type_vocab_size=int(state_dict[b + "embeddings.token_type_embeddings.weight"].shape[0]),
                num_layers=n_layers, num_heads=int(bert_config.num_attention_heads),
                intermediate_size=int(state_dict[b + "encoder.layer.0.intermediate.dense.weight"].shape[0]),
                d_proj=int(args.d_proj), layer_norm_eps=float(bert_config.layer_norm_eps), proj_layer_norm_eps=1e-5)
    return dict(vars(args), bert=bert)


def engine_weights(state_dict, cfg):
    """(audio-tower tensors in agpt_cnn14_create's order, text-tower tensors in agpt_clap_create's order) from a
    checkpoint's "model" dict; a missing key raises KeyError, unused keys are ignored."""
    def pick(keys):
        missing = [k for k in keys if k not in state_dict]
        if missing:
            raise KeyError(f"CLAP checkpoint lacks {missing[:4]}{' ...' if len(missing) > 4 else ''}")
        return [state_dict[k].detach().to("cpu", torch.float32).contiguous() for k in keys]

    return (pick(specs.cnn14_engine_keys(cfg)),
            pick(list(specs.clap_param_shapes(specs.clap_scorer_bert_cfg(cfg)))))


class _Scorer:
    """The two engine handles of one checkpoint: the Cnn14 audio tower and the BERT text tower."""

    def __init__(self, cfg, state_dict, device):
        self.cfg = cfg
        self.device = device
        self.audio_w, self.text_w = engine_weights(state_dict, cfg)
        self.logit_scale = state_dict["logit_scale"].detach().float().cpu() if "logit_scale" in state_dict else None
        self.bert = specs.clap_scorer_bert_cfg(cfg)
        self.audio = _lib.Engine("agpt_cnn14_create")
        acfg = _lib.Cnn14Config(window_size=int(cfg["window_size"]), hop_size=int(cfg["hop_size"]),
                                mel_bins=int(cfg["mel_bins"]), out_emb=int(cfg["out_emb"]), d_proj=int(cfg["d_proj"]))
        self.audio.ensure(device, self.audio_w, lambda: ((C.byref(acfg),), self.audio_w))
        self.text = _lib.Engine("agpt_clap_create")
        tcfg = _lib.ClapConfig(**self.bert)
        self.text.ensure(device, self.text_w, lambda: ((C.byref(tcfg),), self.text_w))
        self._rate = None

    def set_rate(self, sr, resample):
        """The resampler and clip length for input rate sr (resample=False: the clip is used as it is)."""
        key = (int(sr), bool(resample))
        if key == self._rate:
            return
        if resample and int(sr) != int(self.cfg["sampling_rate"]):
            k, width, o, n = specs.sinc_resample_kernel(int(sr), int(self.cfg["sampling_rate"]))
        else:
            k, width, o, n = torch.ones(1, 1), 0, 1, 1
        self._table = np.ascontiguousarray(k.numpy(), dtype=np.float32)
        self._resample = (o, n)
        clip = int(self.cfg["duration"]) * int(sr)
        _lib.check(_lib.lib().agpt_cnn14_set_resample(self.audio.h, o, n, width, self._table.ctypes.data_as(C.c_void_p), clip))
        self._rate, self.clip = key, clip

    def resampled_len(self, L):
        o, n = self._resample
        return (n * L + o - 1) // o


class CLAPWrapper:
    """A class for interfacing CLAP model (wav_evaluation's CLAPWrapper on the engine)."""

    def __init__(self, model_fp, config_path, use_cuda=False):
        self.np_str_obj_array_pattern = re.compile(r"[SaUO]")
        self.file_path = os.path.realpath(__file__)
        with open(config_path, "r") as f:
            self.config_as_str = f.read()
        self.model_fp = model_fp
        self.use_cuda = use_cuda
        if not use_cuda:
            raise RuntimeError("audiogpt_b200.CLAPWrapper runs on CUDA only (use_cuda=True; no CPU fallback)")
        _lib.require_cuda()
        self.clap, self.tokenizer, self.args = self.load_clap()

    def load_clap(self):
        """The engines (cached for one checkpoint, see the module docstring), the tokenizer and the config args."""
        args = read_config_as_args(self.config_as_str, is_config_str=True)
        self.token_keys = ["input_ids", "token_type_ids", "attention_mask"] if "bert" in args.text_model \
            else ["input_ids", "attention_mask"]
        dev = torch.device("cuda", torch.cuda.current_device())
        st = os.stat(self.model_fp)
        key = (os.path.realpath(self.model_fp), st.st_size, st.st_mtime_ns, self.config_as_str, dev.index)
        hit = _CACHE.get(key)
        if hit is None:
            _CACHE.clear()                       # one entry: drop the old engines before building new ones
            sd = torch.load(self.model_fp, map_location=torch.device("cpu"))["model"]
            from transformers import AutoConfig, AutoTokenizer
            cfg = scorer_config(args, sd, AutoConfig.from_pretrained(args.text_model))
            hit = (_Scorer(cfg, sd, dev), AutoTokenizer.from_pretrained(args.text_model))
            _CACHE[key] = hit
        return hit[0], hit[1], args

    @classmethod
    def from_config(cls, cfg, state_dict, tokenizer=None, device=None):
        """Built from a specs.CLAP_SCORER-style config and a checkpoint "model" dict, with no file or hub access and
        no cache."""
        _lib.require_cuda()
        self = cls.__new__(cls)
        self.np_str_obj_array_pattern = re.compile(r"[SaUO]")
        self.file_path = os.path.realpath(__file__)
        self.config_as_str, self.model_fp, self.use_cuda = None, None, True
        self.args = argparse.Namespace(**{k: v for k, v in cfg.items() if k != "bert"})
        self.token_keys = ["input_ids", "token_type_ids", "attention_mask"]
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.clap = _Scorer(dict(cfg), state_dict, dev)
        self.tokenizer = tokenizer
        return self

    # ------------------------------------------------------------------ text
    def preprocess_text(self, text_queries):
        """Tokenize each query as the reference does (encode_plus, max_length=text_len, padding to it, no truncation)
        and stack the rows: {key: [N, L]} on the host."""
        if self.tokenizer is None:
            raise RuntimeError("audiogpt_b200.CLAPWrapper: no tokenizer (use encode_text_ids)")
        rows = []
        for t in text_queries:
            tok = self.tokenizer.encode_plus(text=t, add_special_tokens=True, max_length=self.args.text_len,
                                             padding="max_length", return_tensors="pt")
            rows.append({k: torch.as_tensor(tok[k]).reshape(-1) for k in self.token_keys})
        lens = {r["input_ids"].shape[0] for r in rows}
        if len(lens) != 1:
            raise RuntimeError("each element in list of batch should be of equal size")
        return {k: torch.stack([r[k] for r in rows]) for k in self.token_keys}

    @torch.no_grad()
    def encode_text_ids(self, input_ids, token_type_ids=None, attention_mask=None):
        """[N, L] integer CUDA tensors -> the normalised text embeddings [N, d_proj] (the tokenizer-free entry)."""
        if not input_ids.is_cuda:
            raise RuntimeError("audiogpt_b200.CLAPWrapper runs on CUDA only (no CPU fallback)")
        if input_ids.dim() != 2 or input_ids.is_floating_point():
            raise ValueError(f"input_ids must be an integer [N, L] tensor, got {input_ids.dtype} {tuple(input_ids.shape)}")
        N, L = input_ids.shape
        b = self.clap.bert
        if N < 1 or L < 1:
            raise ValueError(f"empty input_ids {tuple(input_ids.shape)}")
        if L > b["max_position_embeddings"]:
            raise ValueError(f"sequence length {L} > max_position_embeddings {b['max_position_embeddings']}")
        token_type_ids = torch.zeros_like(input_ids) if token_type_ids is None else token_type_ids
        attention_mask = torch.ones_like(input_ids) if attention_mask is None else attention_mask
        for name, t, hi in (("token ids", input_ids, b["vocab_size"]), ("token type ids", token_type_ids, b["type_vocab_size"])):
            if t.shape != input_ids.shape or not t.is_cuda:
                raise ValueError(f"{name} must be a CUDA tensor of shape {tuple(input_ids.shape)}")
            lo_, hi_ = (int(v) for v in torch.aminmax(t))
            if lo_ < 0 or hi_ >= hi:
                raise ValueError(f"{name} must lie in [0, {hi}), got [{lo_}, {hi_}]")
        if attention_mask.shape != input_ids.shape or not attention_mask.is_cuda:
            raise ValueError(f"attention_mask must be a CUDA tensor of shape {tuple(input_ids.shape)}")
        dev = input_ids.device
        ids, tys, msk = (t.to(torch.int32).contiguous() for t in (input_ids, token_type_ids, attention_mask))
        out = torch.empty((N, b["d_proj"]), device=dev, dtype=torch.float32)
        self.clap.text.call("clap_encode_cls", dev, _lib.fptr(ids), _lib.fptr(tys), _lib.fptr(msk), N, L, _lib.fptr(out))
        return out

    def get_text_embeddings(self, class_labels):
        r"""Load list of class labels and return text embeddings"""
        tok = self.preprocess_text(class_labels)
        dev = self.clap.device
        return self.encode_text_ids(*(tok[k].to(dev) if k in tok else None
                                      for k in ("input_ids", "token_type_ids", "attention_mask")))

    # ------------------------------------------------------------------ audio
    def _clip_of(self, audio_file):
        if isinstance(audio_file, str):
            import torchaudio
            wav, sr = torchaudio.load(audio_file)
        elif isinstance(audio_file, tuple):
            wav, sr = audio_file
        else:
            raise TypeError(f"type of audiofile is {type(audio_file)},which is not supported")
        wav = torch.as_tensor(wav)
        if wav.dim() > 1 and wav.shape[0] != 1 or wav.dim() > 2:
            raise ValueError(f"audiogpt_b200.CLAPWrapper takes mono clips, got shape {tuple(wav.shape)}")
        return wav.reshape(-1), int(sr)

    @torch.no_grad()
    def embed_audio(self, wav, sr, starts, resample=True):
        """wav [B, n] CUDA float clips at rate sr, starts: per clip the crop start drawn for it or -1 (tile) ->
        the normalised audio embeddings [B, d_proj]."""
        if not wav.is_cuda:
            raise RuntimeError("audiogpt_b200.CLAPWrapper runs on CUDA only (no CPU fallback)")
        if wav.dim() != 2 or wav.shape[0] < 1 or wav.shape[1] < 1:
            raise ValueError(f"wav must be [B, n], got {tuple(wav.shape)}")
        B = wav.shape[0]
        self.clap.set_rate(sr, resample)
        x = wav.to(torch.float32).contiguous()
        st = (C.c_int * B)(*[int(s) for s in starts])
        out = torch.empty((B, int(self.clap.cfg["d_proj"])), device=wav.device, dtype=torch.float32)
        self.clap.audio.call("cnn14_embed", wav.device, _lib.fptr(x), int(wav.shape[1]), B, st, _lib.fptr(out))
        return out

    def get_audio_embeddings(self, audio_files, resample):
        r"""Load list of audio files and return a audio embeddings"""
        dev = self.clap.device
        clips = [self._clip_of(a) for a in audio_files]
        starts = []
        for wav, sr in clips:    # the reference's random.randrange draws: one per cropped clip, in list order
            self.clap.set_rate(sr, resample)
            R = self.clap.resampled_len(wav.shape[0])
            starts.append(-1 if self.clap.clip >= R else random.randrange(R - self.clap.clip))
        if len({(w.shape[0], sr) for w, sr in clips}) == 1:
            return self.embed_audio(torch.stack([w for w, _ in clips]).to(dev), clips[0][1], starts, resample)
        return torch.cat([self.embed_audio(w[None].to(dev), sr, [s], resample) for (w, sr), s in zip(clips, starts)])

    # ------------------------------------------------------------------ scores
    @torch.no_grad()
    def compute_similarity(self, audio_embeddings, text_embeddings, use_logit_scale=True):
        r"""Compute similarity between text and audio embeddings: (t @ a.T).T, [N_audio, N_text]"""
        a, t = audio_embeddings.float().contiguous(), text_embeddings.float().contiguous()
        if not (a.is_cuda and t.is_cuda):
            raise RuntimeError("audiogpt_b200.CLAPWrapper runs on CUDA only (no CPU fallback)")
        if a.dim() != 2 or t.dim() != 2 or a.shape[1] != t.shape[1]:
            raise ValueError(f"embeddings must be [N, D] with one D, got {tuple(a.shape)} and {tuple(t.shape)}")
        scale = 1.0
        if use_logit_scale:
            if self.clap.logit_scale is None:
                raise KeyError("the checkpoint has no logit_scale")
            scale = math.exp(float(self.clap.logit_scale))
        out = torch.empty((a.shape[0], t.shape[0]), device=a.device, dtype=torch.float32)
        with torch.cuda.device(a.device):
            _lib.check(_lib.lib().agpt_clap_similarity(_lib.fptr(a), a.shape[0], _lib.fptr(t), t.shape[0], a.shape[1],
                                                       scale, _lib.fptr(out), _lib.cur_stream(a.device)))
        return out

    def cal_clap_score(self, txt, audio_path):
        text_embeddings = self.get_text_embeddings([txt])
        audio_embeddings = self.get_audio_embeddings([audio_path], resample=True)
        return self.compute_similarity(audio_embeddings, text_embeddings, use_logit_scale=False).squeeze().cpu().numpy()

"""audiogpt_b200 -- H100 (sm_90a) back-end for AudioGPT's generative hot path.

Drop-in classes (same names / signatures / state-dict layouts as the reference):

    audiogpt_b200.modules.hifigan.hifigan.HifiGanGenerator
    audiogpt_b200.vocoders.hifigan.HifiGAN
    audiogpt_b200.modules.diff.net.DiffNet
    audiogpt_b200.modules.diff.shallow_diffusion_tts.GaussianDiffusion
    audiogpt_b200.ldm.modules.diffusionmodules.openaimodel.UNetModel
    audiogpt_b200.ldm.models.diffusion.ddim.DDIMSampler
    audiogpt_b200.ldm.models.autoencoder.AutoencoderKL          (decode side; not installed over the reference class)
    audiogpt_b200.ldm.models.autoencoder.AutoencoderKLWithEncoder   (whole first stage; installed as AutoencoderKL
                                                                     with install(first_stage=True))
    audiogpt_b200.modules.fastspeech.pe.PitchExtractor
    audiogpt_b200.vocoder.bigvgan.models.BigVGAN / VocoderBigVGAN
    audiogpt_b200.modules.fastspeech.fs2.FastSpeech2                (installed with install(front_end=True))
    audiogpt_b200.modules.diffsinger_midi.fs2.FastSpeech2MIDI       (installed with install(front_end=True))
    audiogpt_b200.ldm.modules.encoders.modules.FrozenCLAPEmbedder   (installed with install(text_encoder=True))
    audiogpt_b200.wav_evaluation.models.CLAPWrapper.CLAPWrapper     (installed with install(scorer=True))
    audiogpt_b200.modules.GenerSpeech.model.generspeech.GenerSpeech (installed with install(tts_ood=True))
    audiogpt_b200.sound_extraction.model.LASSNet.LASSNet            (installed with install(extraction=True))
    audiogpt_b200.sound_extraction.utils.stft.STFT                  (installed with install(extraction=True))
    audiogpt_b200.audio_detection.audio_infer.pytorch.models.PVT    (installed with install(detection=True))
    audiogpt_b200.audio_detection.target_sound_detection.src.models.RaDur_fusion
                                                                    (installed with install(target_detection=True))
    audiogpt_b200.mono2binaural.src.models.BinauralNetwork          (installed with install(binaural=True))
    audiogpt_b200.inference.tts.base_tts_infer.Wav2Vec2ForCTC       (installed with install(asr=True))
    audiogpt_b200.data_gen.tts.emotion.model.EmotionEncoder         (installed with install(emotion=True))
    audiogpt_b200.data_gen.tts.emotion.inference.embed_utterance / embed_frames_batch
                                                                    (installed with install(emotion=True))

All arithmetic lives in libagpt_b200.so (audiogpt_b200/csrc, C ABI in include/agpt_b200.h).
There is no CPU fallback.
"""
__version__ = "0.1.0"

# reference module name -> (our module, attributes to graft onto the reference module: a list of names, or a
# {reference name: our name} mapping)
_INSTALL_MAP = {
    "modules.hifigan.hifigan": ("audiogpt_b200.modules.hifigan.hifigan", ["HifiGanGenerator"]),
    "vocoders.hifigan": ("audiogpt_b200.vocoders.hifigan", ["HifiGAN", "load_model"]),
    "modules.diff.net": ("audiogpt_b200.modules.diff.net", ["DiffNet"]),
    "modules.diff.shallow_diffusion_tts": ("audiogpt_b200.modules.diff.shallow_diffusion_tts",
                                           ["GaussianDiffusion", "noise_like"]),
    "ldm.modules.diffusionmodules.openaimodel": ("audiogpt_b200.ldm.modules.diffusionmodules.openaimodel",
                                                 ["UNetModel"]),
    "ldm.models.diffusion.ddim": ("audiogpt_b200.ldm.models.diffusion.ddim", ["DDIMSampler"]),
    "vocoder.bigvgan.models": ("audiogpt_b200.vocoder.bigvgan.models", ["BigVGAN", "VocoderBigVGAN"]),
    "modules.fastspeech.pe": ("audiogpt_b200.modules.fastspeech.pe", ["PitchExtractor"]),
}
# the acoustic front-end, grafted only on request (install(front_end=True))
_FRONT_END_MAP = {
    "modules.fastspeech.fs2": ("audiogpt_b200.modules.fastspeech.fs2", ["FastSpeech2"]),
    "modules.diffsinger_midi.fs2": ("audiogpt_b200.modules.diffsinger_midi.fs2", ["FastSpeech2MIDI"]),
}
# the whole first stage of the Make-An-Audio tools, grafted only on request (install(first_stage=True))
_FIRST_STAGE_MAP = {
    "ldm.models.autoencoder": ("audiogpt_b200.ldm.models.autoencoder", {"AutoencoderKL": "AutoencoderKLWithEncoder"}),
}
# the CLAP text encoder of the Make-An-Audio tools, grafted only on request (install(text_encoder=True))
_TEXT_ENCODER_MAP = {
    "ldm.modules.encoders.modules": ("audiogpt_b200.ldm.modules.encoders.modules", ["FrozenCLAPEmbedder"]),
}
# the CLAP candidate scorer of the text-to-audio tool, grafted only on request (install(scorer=True)); the reference
# module does not import on torch 2.x, so outside strict mode this is the sys.modules alias
_SCORER_MAP = {
    "wav_evaluation.models.CLAPWrapper": ("audiogpt_b200.wav_evaluation.models.CLAPWrapper", ["CLAPWrapper"]),
}

# the out-of-domain TTS tool's acoustic model, grafted only on request (install(tts_ood=True))
_TTS_OOD_MAP = {
    "modules.GenerSpeech.model.generspeech": ("audiogpt_b200.modules.GenerSpeech.model.generspeech", ["GenerSpeech"]),
}

# the sound-extraction tool's network and STFT, grafted only on request (install(extraction=True))
_EXTRACTION_MAP = {
    "sound_extraction.model.LASSNet": ("audiogpt_b200.sound_extraction.model.LASSNet", ["LASSNet"]),
    "sound_extraction.utils.stft": ("audiogpt_b200.sound_extraction.utils.stft", ["STFT"]),
}

# the sound-event-detection tool's PVT, grafted only on request (install(detection=True)) under the name the agent
# script imports at load time (audio_detection/ is on its sys.path); the reference module imports torchlibrosa, timm,
# mmcv and mmdet, so where those are missing this is the sys.modules alias
_DETECTION_MAP = {
    "audio_infer.pytorch.models": ("audiogpt_b200.audio_detection.audio_infer.pytorch.models", ["PVT"]),
}

# the target-sound-detection tool's RaDur_fusion, grafted only on request (install(target_detection=True)).  The tool
# also imports the reference module's event_labels, so the module is patched in place and never aliased: when it does
# not import, the name is reported as skipped.
_TARGET_DETECTION_MAP = {
    "target_sound_detection.src.models": ("audiogpt_b200.audio_detection.target_sound_detection.src.models", ["RaDur_fusion"]),
}

# the TTS_OOD tool's reference-audio ASR, grafted only on request (install(asr=True)).  The module also holds
# BaseTTSInfer, which the TTS inferers import, so it is patched in place as _TARGET_DETECTION_MAP is, never aliased.
_ASR_MAP = {
    "inference.tts.base_tts_infer": ("audiogpt_b200.inference.tts.base_tts_infer", ["Wav2Vec2ForCTC"]),
}

# the TTS_OOD tool's emotion encoder, grafted only on request (install(emotion=True)).  The inference module also holds
# preprocess_wav and load_model, which stay the reference's, so both modules are patched in place, never aliased.
_EMOTION_MAP = {
    "data_gen.tts.emotion.model": ("audiogpt_b200.data_gen.tts.emotion.model", ["EmotionEncoder"]),
    "data_gen.tts.emotion.inference": ("audiogpt_b200.data_gen.tts.emotion.inference",
                                       ["EmotionEncoder", "embed_frames_batch", "embed_utterance"]),
}

# the Binaural tool's BinauralNetwork, grafted only on request (install(binaural=True)).  The tool imports it as
# ``src.models`` (mono2binaural/ on its sys.path), a generic name: the module is patched in place only when it is the
# reference's (it defines Warpnet and BinauralNetwork), and never aliased.
_BINAURAL_MAP = {
    "src.models": ("audiogpt_b200.mono2binaural.src.models", ["BinauralNetwork"]),
}


def install(strict: bool = False, front_end: bool = False, first_stage: bool = False, inpaint: bool = False,
            text_encoder: bool = False, scorer: bool = False, tts_ood: bool = False, extraction: bool = False, detection: bool = False,
            target_detection: bool = False, binaural: bool = False, asr: bool = False, emotion: bool = False):
    """Make AudioGPT's tool classes pick up this back-end.

    Call once, after the reference's packages are importable (``sys.path`` contains
    ``NeuralSeq/`` and ``text_to_audio/Make_An_Audio/``) and before ``audio-chatgpt.py`` builds its
    tools.  For every reference module that is importable, the hot-path classes are replaced in
    place (``setattr`` on the reference module), so ``from modules.hifigan.hifigan import
    HifiGanGenerator``, ``instantiate_from_config({'target':
    'ldm.modules.diffusionmodules.openaimodel.UNetModel', ...})`` and ``DDIMSampler(model)`` all
    resolve to the drop-ins.  Modules that are not importable are registered in ``sys.modules``
    as aliases of ours when ``strict`` is False.  ``front_end=True`` also replaces FastSpeech2 and
    FastSpeech2MIDI, so GaussianDiffusion's front-end (and any other user of those classes) runs on the engine.
    ``first_stage=True`` also replaces ``ldm.models.autoencoder.AutoencoderKL`` by AutoencoderKLWithEncoder, so
    every Make-An-Audio tool encodes and decodes its first stage on the engine, and records the reference's
    DiagonalGaussianDistribution as the class its encode() returns.
    ``inpaint=True`` also makes ``UNetModel(...)`` build AttentionUNetModel for the AttentionBlock configs it covers
    (the Inpaint tool's denoiser) instead of the reference's class, so with ``first_stage=True`` the whole Inpaint
    chain runs on the engine.
    ``text_encoder=True`` also replaces ``ldm.modules.encoders.modules.FrozenCLAPEmbedder``, so the text-to-audio tool's
    conditioning (get_learned_conditioning) runs on the engine too, from token ids to waveform.
    ``scorer=True`` also replaces ``wav_evaluation.models.CLAPWrapper.CLAPWrapper``, so the import inside
    T2A.select_best_audio resolves to the drop-in and the candidate scoring runs on the engine.
    ``tts_ood=True`` also replaces ``modules.GenerSpeech.model.generspeech.GenerSpeech``, so the import in
    inference/tts/GenerSpeech.py resolves to the drop-in and the TTS_OOD tool's acoustic model and post-flow run on the
    engine (its HiFi-GAN vocoder is grafted by default).
    ``extraction=True`` also replaces ``sound_extraction.model.LASSNet.LASSNet`` and ``sound_extraction.utils.stft.STFT``,
    so the SoundExtraction tool's STFT, text encoder, FiLM ResUNet and inverse STFT run on the engine.
    ``detection=True`` also replaces ``audio_infer.pytorch.models.PVT``, so the SoundDetection tool's log-mel front end,
    pyramid transformer and framewise head run on the engine.  The agent script imports that name when it is loaded, so
    call install first; only the ``models`` leaf is aliased, the packages ``audio_infer`` and ``audio_infer.pytorch``
    (from which the script also imports ``audio_infer.utils.config``) stay the reference's own.
    ``target_detection=True`` also replaces ``target_sound_detection.src.models.RaDur_fusion``, so the TargetSoundDetection
    tool's Cnn14 reference encoder, multi-scale CNN, bidirectional GRU and enhancement pass run on the engine.  That
    module is only patched in place: the tool also imports its ``event_labels``, so when it does not import it is
    reported as skipped (and raises under ``strict``), never aliased.
    ``asr=True`` also replaces ``inference.tts.base_tts_infer.Wav2Vec2ForCTC``, so build_asr's
    ``Wav2Vec2ForCTC.from_pretrained`` builds the drop-in and the TTS_OOD tool's reference-audio transcription runs on the
    engine.  Like ``target_detection``, the module is only patched in place (it also holds BaseTTSInfer): when it does not
    import it is reported as skipped (and raises under ``strict``), never aliased.
    ``emotion=True`` also replaces ``data_gen.tts.emotion.model.EmotionEncoder`` and, in
    ``data_gen.tts.emotion.inference``, ``EmotionEncoder``, ``embed_frames_batch`` and ``embed_utterance``: the reference's
    load_model then builds the drop-in, and the TTS_OOD tool's emo_embed runs on the engine.  inference/tts/GenerSpeech.py
    binds ``embed_utterance`` by name when it is imported, so call install before that module is loaded (when it already
    is, its ``Embed_utterance`` is rebound too).  Like ``asr``, the modules are only patched in place: when one does not
    import (it needs webrtcvad, librosa and matplotlib) it is reported as skipped (and raises under ``strict``).
    ``binaural=True`` also replaces ``src.models.BinauralNetwork`` (mono2binaural/src/models.py), so the Binaural tool's
    geometric and neural time warp run on the engine.  ``src`` is a generic name, so the module is patched in place only
    when it is the reference's (it defines ``Warpnet`` and ``BinauralNetwork``); when it does not import or is some other
    ``src``, it is reported as skipped (and raises under ``strict``), never aliased.
    Returns the list of patched names."""
    import importlib
    import sys
    import types
    patched = []
    todo = dict(_INSTALL_MAP, **(_FRONT_END_MAP if front_end else {}), **(_FIRST_STAGE_MAP if first_stage else {}),
                **(_TEXT_ENCODER_MAP if text_encoder else {}), **(_SCORER_MAP if scorer else {}),
                **(_TTS_OOD_MAP if tts_ood else {}), **(_EXTRACTION_MAP if extraction else {}), **(_DETECTION_MAP if detection else {}))
    for ref_name, (our_name, attrs) in todo.items():
        ours = importlib.import_module(our_name)
        names = attrs if isinstance(attrs, dict) else {a: a for a in attrs}
        try:
            ref = importlib.import_module(ref_name)
        except Exception:
            if strict:
                raise
            alias = ours
            if any(a != b for a, b in names.items()):
                # a renamed graft: the alias is a copy of our module with the reference's names bound to our classes
                alias = types.ModuleType(ref_name, ours.__doc__)
                alias.__dict__.update({k: v for k, v in vars(ours).items() if not k.startswith("__")})
                for a, b in names.items():
                    setattr(alias, a, getattr(ours, b))
            sys.modules.setdefault(ref_name, alias)
            patched.append(ref_name + " (aliased)")
            continue
        for a, b in names.items():
            theirs = getattr(ref, a, None)
            mine = getattr(ours, b)
            # configs the drop-in does not cover (e.g. the inpainting AttentionBlock UNet) keep the reference class
            if hasattr(mine, "_reference_cls") and isinstance(theirs, type) and theirs is not mine:
                mine._reference_cls = theirs
            setattr(ref, a, mine)
        patched.append(ref_name)
    in_place = dict(**(_TARGET_DETECTION_MAP if target_detection else {}), **(_ASR_MAP if asr else {}),
                    **(_EMOTION_MAP if emotion else {}))
    if in_place:
        for ref_name, (our_name, attrs) in in_place.items():
            ours = importlib.import_module(our_name)
            try:
                ref = importlib.import_module(ref_name)
            except Exception:
                if strict:
                    raise
                patched.append(ref_name + " (skipped: not importable)")
                continue
            for a in attrs:
                setattr(ref, a, getattr(ours, a))
            if ref_name == "data_gen.tts.emotion.inference":
                ours._state = ref    # the reference's load_model stores the model there
                tool = sys.modules.get("inference.tts.GenerSpeech")
                if tool is not None:
                    tool.Embed_utterance = ours.embed_utterance
            patched.append(ref_name)
    if binaural:
        for ref_name, (our_name, attrs) in _BINAURAL_MAP.items():
            ours = importlib.import_module(our_name)
            try:
                ref = importlib.import_module(ref_name)
            except Exception:
                if strict:
                    raise
                patched.append(ref_name + " (skipped: not importable)")
                continue
            if not all(isinstance(getattr(ref, n, None), type) for n in ("Warpnet", "BinauralNetwork")):
                if strict:
                    raise ImportError(f"{ref_name} ({getattr(ref, '__file__', None)}) is not mono2binaural's: it lacks "
                                      "Warpnet / BinauralNetwork")
                patched.append(ref_name + " (skipped: not mono2binaural's)")
                continue
            for a in attrs:
                setattr(ref, a, getattr(ours, a))
            patched.append(ref_name)
    if inpaint:
        from .ldm.modules.diffusionmodules.openaimodel import AttentionUNetModel, UNetModel
        UNetModel._attention_cls = AttentionUNetModel
        patched.append("ldm.modules.diffusionmodules.openaimodel (AttentionBlock UNets)")
    if first_stage:
        # get_first_stage_encoding checks isinstance(posterior, DiagonalGaussianDistribution) against the reference's
        # own class (ddpm_audio.py:157-164): encode() must build that class when it exists
        try:
            dist = importlib.import_module("ldm.modules.distributions.distributions")
            from .ldm.models.autoencoder import AutoencoderKLWithEncoder
            AutoencoderKLWithEncoder._posterior_cls = dist.DiagonalGaussianDistribution
        except Exception:
            if strict:
                raise
    # the vocoder registry of the reference keeps its own dict: register ours there too
    try:
        bv = importlib.import_module("vocoders.base_vocoder")
        from .vocoders.hifigan import HifiGAN
        bv.VOCODERS["hifigan"] = HifiGAN
        bv.VOCODERS["HifiGAN"] = HifiGAN
    except Exception:
        pass
    return patched

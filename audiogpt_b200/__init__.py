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


def install(strict: bool = False, front_end: bool = False, first_stage: bool = False, inpaint: bool = False,
            text_encoder: bool = False, scorer: bool = False):
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
    Returns the list of patched names."""
    import importlib
    import sys
    import types
    patched = []
    todo = dict(_INSTALL_MAP, **(_FRONT_END_MAP if front_end else {}), **(_FIRST_STAGE_MAP if first_stage else {}),
                **(_TEXT_ENCODER_MAP if text_encoder else {}), **(_SCORER_MAP if scorer else {}))
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

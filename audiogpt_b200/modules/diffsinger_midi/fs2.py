"""Drop-in for ``modules.diffsinger_midi.fs2.FastSpeech2MIDI`` (the text-to-singing front-end).

Reference: /root/reference/NeuralSeq/modules/diffsinger_midi/fs2.py:11-118: FastSpeech2 whose encoder input adds
``midi_embed[pitch_midi] + midi_dur_layer(midi_dur) + is_slur_embed[is_slur]`` to the scaled token embedding
(forward(..., pitch_midi=..., midi_dur=..., is_slur=...)).  Everything else is audiogpt_b200.modules.fastspeech.fs2.
"""
from __future__ import annotations

from ..fastspeech.fs2 import FastSpeech2


class FastSpeech2MIDI(FastSpeech2):
    _use_midi = True

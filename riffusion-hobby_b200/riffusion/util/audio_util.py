"""Audio helpers (reference: riffusion/util/audio_util.py).

pydub is used when it is installed; otherwise the numpy AudioSegment stand-in from
`audio_segment.py` is (pydub/ffmpeg are absent from the GPU image).
"""
from __future__ import annotations

import functools
import io
import typing as T

import numpy as np
from scipy.io import wavfile

try:  # pragma: no cover - depends on the environment
    import pydub
    import pydub.effects

    AudioSegment = pydub.AudioSegment
    _normalize = pydub.effects.normalize
    HAVE_PYDUB = True
except ImportError:  # pragma: no cover
    from riffusion.util.audio_segment import AudioSegment, normalize as _normalize

    pydub = None
    HAVE_PYDUB = False


def int16_from_waveform(samples: np.ndarray, normalize: bool = False) -> np.ndarray:
    """(channels, samples) float -> (samples, channels) int16, audio_util.py:22-28:
    peak-normalise over all channels jointly to int16 max (in place, like the reference) and
    truncate toward zero."""
    if normalize:
        samples *= np.iinfo(np.int16).max / np.max(np.abs(samples))
    return samples.transpose(1, 0).astype(np.int16)


def audio_from_waveform(samples: np.ndarray, sample_rate: int, normalize: bool = False):
    """(channels, samples) float waveform -> AudioSegment via an in-memory WAV."""
    pcm = int16_from_waveform(samples, normalize=normalize)
    wav_bytes = io.BytesIO()
    wavfile.write(wav_bytes, sample_rate, pcm)
    wav_bytes.seek(0)
    return AudioSegment.from_wav(wav_bytes)


_TARGET_DBFS = -12.0          # loudness every clip is brought to before the final peak normalisation
_PEAK_HEADROOM_DB = 0.1


def apply_filters(segment, compression: bool = False):
    """Loudness post-processing of a reconstructed clip (audio_util.py:39-72): optional dynamic-range compression (pydub
    only), then gain to -12 dBFS and a peak normalisation that leaves 0.1 dB of headroom."""
    if compression:
        if not HAVE_PYDUB:
            raise NotImplementedError("compress_dynamic_range needs pydub (not installed)")
        levelled = _normalize(segment, headroom=_PEAK_HEADROOM_DB)
        levelled = levelled.apply_gain(-10 - levelled.dBFS)
        segment = pydub.effects.compress_dynamic_range(levelled, threshold=-20.0, ratio=4.0, attack=5.0, release=50.0)
    at_target = segment.apply_gain(_TARGET_DBFS - segment.dBFS)
    return _normalize(at_target, headroom=_PEAK_HEADROOM_DB)


def stitch_segments(segments: T.Sequence, crossfade_s: float):
    """Play the segments one after another, blending each junction over `crossfade_s` seconds (audio_util.py:75-85)."""
    fade_ms = int(crossfade_s * 1000)
    return functools.reduce(lambda so_far, nxt: so_far.append(nxt, crossfade=fade_ms), segments[1:], segments[0])


def overlay_segments(segments: T.Sequence):
    """Mix all segments on top of the first one (audio_util.py:88-99)."""
    assert len(segments) > 0
    return functools.reduce(lambda mix, nxt: mix.overlay(nxt), segments[1:], segments[0])

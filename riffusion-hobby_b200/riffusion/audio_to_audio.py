"""Host-side bookkeeping of the audio-to-audio task (riffusion/streamlit/tasks/audio_to_audio.py): which clips a track is
cut into, and the image size the clips are denoised at.  The numpy expressions are the reference's, float quirks
included (a clip starting at 14.4 s is cut at 14399 ms).  `RiffusionPipeline.audio_to_audio` runs the task on the device.
"""
from __future__ import annotations

import typing as T

import numpy as np

from riffusion.util.audio_util import AudioSegment


def clip_start_times(track_duration_s: float, start_time_s: float = 0.0, duration_s: float = 20.0,
                     clip_duration_s: float = 5.0, overlap_duration_s: float = 0.2) -> np.ndarray:
    """Start times (s) of the overlapping clips (audio_to_audio.py:99-101): the requested duration is cut to what the
    track holds after `start_time_s`, and a clip starts every clip_duration_s - overlap_duration_s seconds."""
    duration_s = min(duration_s, track_duration_s - start_time_s)
    increment_s = clip_duration_s - overlap_duration_s
    return start_time_s + np.arange(0, duration_s - clip_duration_s, increment_s)


def slice_audio_into_clips(segment, clip_starts: T.Sequence[float], clip_duration_s: float) -> T.List:
    """The clips [int(s * 1000), int(s * 1000) + int(clip_duration_s * 1000)) ms of `segment`; the last one is padded
    with silence if it is short (audio_to_audio.py:396-416).  The silence is made at the clip's frame rate and appended
    without a crossfade: the reference's pydub call would resample 11025 Hz silence and crossfade 100 ms into it, which
    fails for padding under 100 ms.  Start times from `clip_start_times` never need padding."""
    clips = []
    for i, start_s in enumerate(clip_starts):
        start_ms = int(start_s * 1000)
        clip_ms = int(clip_duration_s * 1000)
        clip = segment[start_ms:start_ms + clip_ms]
        if i == len(clip_starts) - 1:
            silence_ms = clip_ms - int(clip.duration_seconds * 1000)
            if silence_ms > 0:
                clip = clip.append(AudioSegment.silent(duration=silence_ms, frame_rate=clip.frame_rate), crossfade=0)
        clips.append(clip)
    return clips


def stride_32_size(width: int, height: int) -> T.Tuple[int, int]:
    """The size `scale_image_to_32_stride` (audio_to_audio.py:419-425) resizes a clip image to: each side rounded up to
    a multiple of 32."""
    return int(np.ceil(width / 32) * 32), int(np.ceil(height / 32) * 32)


def check_denoising_size(width: int, height: int, clip_duration_s: float) -> None:
    """The UNet of this package takes latents whose sides are multiples of 8, i.e. images whose sides are multiples of
    64; diffusers would upsample odd latent sizes instead (forward_upsample_size), which is not implemented."""
    if width % 64 or height % 64:
        raise ValueError(
            f"a {clip_duration_s} s clip gives a {width}x{height} image after rounding up to a 32-pixel stride; the "
            "denoiser needs multiples of 64.  Among whole-second clip durations 3, 5, 7, 8 and 10 s work and 4, 6 and "
            "9 s do not")


def clip_frames(clip_duration_s: float, sample_rate: int, hop_length: int) -> int:
    """Spectrogram columns of one clip of int(clip_duration_s * 1000) ms: 1 + samples // hop."""
    samples = int(int(clip_duration_s * 1000) * sample_rate / 1000.0)
    return 1 + samples // hop_length

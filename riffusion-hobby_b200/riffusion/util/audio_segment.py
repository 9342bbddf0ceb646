"""Minimal numpy-backed stand-in for pydub.AudioSegment.

pydub (and ffmpeg) are not installed in the GPU image, but the reference API passes
`pydub.AudioSegment` objects across `SpectrogramConverter.spectrogram_from_audio` /
`audio_from_spectrogram` (spectrogram_converter.py:101-163).  When pydub is importable it is
used; otherwise this class provides the subset of its surface the converter, the image
converter, audio_util and the CLI touch — WAV only, integer PCM.

Semantics restated from pydub 0.25 [memory, package absent here — parity unpinned]:
  * samples are interleaved little-endian signed ints of `sample_width` bytes;
  * `len(seg)` is the duration in ms, `seg[a:b]` slices in ms;
  * `rms` = int(sqrt(mean(x^2))) (audioop.rms), `dBFS` = 20 log10(rms / max_possible_amplitude);
  * `apply_gain(db)` multiplies by 10^(db/20), floors and clips (audioop.mul);
  * `set_channels(1)` averages the two channels with floor division (audioop.tomono 0.5/0.5);
    `set_channels(2)` on mono duplicates the channel.
"""
from __future__ import annotations

import array
import io
import math
import typing as T

import numpy as np
from scipy.io import wavfile

_DTYPES = {1: np.int8, 2: np.int16, 4: np.int32}


def db_to_float(db: float) -> float:
    return 10 ** (float(db) / 20)


def ratio_to_db(ratio: float) -> float:
    if ratio == 0:
        return -float("inf")
    return 20 * math.log10(ratio)


class AudioSegment:
    def __init__(self, samples: np.ndarray, frame_rate: int):
        """samples: (frames, channels) integer array."""
        samples = np.asarray(samples)
        if samples.ndim == 1:
            samples = samples[:, None]
        if samples.dtype not in (np.int8, np.int16, np.int32):
            raise TypeError(f"unsupported sample dtype {samples.dtype}")
        self._s = np.ascontiguousarray(samples)
        self.frame_rate = int(frame_rate)

    # ---- constructors / io
    @classmethod
    def from_wav(cls, file) -> "AudioSegment":
        rate, data = wavfile.read(file)
        if data.dtype == np.uint8:  # 8-bit WAV is unsigned
            data = (data.astype(np.int16) - 128).astype(np.int8)
        if data.dtype.kind == "f":
            raise TypeError("float WAV files are not supported by the AudioSegment stand-in")
        return cls(data, rate)

    @classmethod
    def from_file(cls, file, format: T.Optional[str] = None) -> "AudioSegment":
        name = str(file)
        if (format or name.rsplit(".", 1)[-1]).lower() not in ("wav", "wave"):
            raise NotImplementedError(
                "only WAV files can be read without pydub/ffmpeg (not installed in this image)")
        return cls.from_wav(file)

    @classmethod
    def silent(cls, duration: int = 1000, frame_rate: int = 11025) -> "AudioSegment":
        return cls(np.zeros((int(frame_rate * duration / 1000.0), 1), np.int16), frame_rate)

    def export(self, out_f=None, format: str = "wav", **_kw):
        if format.lower() not in ("wav", "wave"):
            raise NotImplementedError("only WAV export is available without pydub/ffmpeg")
        data = self._s if self.channels > 1 else self._s[:, 0]
        if out_f is None:
            out_f = io.BytesIO()
        wavfile.write(out_f, self.frame_rate, data)
        if hasattr(out_f, "seek"):
            out_f.seek(0)
        return out_f

    # ---- properties
    @property
    def channels(self) -> int:
        return int(self._s.shape[1])

    @property
    def sample_width(self) -> int:
        return int(self._s.dtype.itemsize)

    @property
    def frame_width(self) -> int:
        return self.channels * self.sample_width

    @property
    def raw_data(self) -> bytes:
        return self._s.tobytes()

    def frame_count(self) -> float:
        return float(self._s.shape[0])

    @property
    def duration_seconds(self) -> float:
        return self._s.shape[0] / self.frame_rate if self.frame_rate else 0.0

    def __len__(self) -> int:
        return round(1000 * (self.frame_count() / self.frame_rate))

    @property
    def max_possible_amplitude(self) -> float:
        return (2 ** (self.sample_width * 8)) / 2

    @property
    def max(self) -> int:
        return int(np.abs(self._s.astype(np.int64)).max()) if self._s.size else 0

    @property
    def rms(self) -> int:
        if not self._s.size:
            return 0
        x = self._s.astype(np.float64).ravel()
        return int(math.sqrt(float(np.dot(x, x)) / x.size))

    @property
    def dBFS(self) -> float:
        rms = self.rms
        if not rms:
            return -float("inf")
        return ratio_to_db(rms / self.max_possible_amplitude)

    # ---- sample access
    def get_array_of_samples(self) -> array.array:
        code = {1: "b", 2: "h", 4: "i"}[self.sample_width]
        return array.array(code, self._s.ravel().tobytes())

    def split_to_mono(self) -> T.List["AudioSegment"]:
        return [AudioSegment(self._s[:, c : c + 1].copy(), self.frame_rate) for c in range(self.channels)]

    def set_channels(self, channels: int) -> "AudioSegment":
        if channels == self.channels:
            return self
        if channels == 2 and self.channels == 1:
            return AudioSegment(np.repeat(self._s, 2, axis=1), self.frame_rate)
        if channels == 1 and self.channels == 2:
            # audioop.tomono(data, width, 0.5, 0.5): floor(l*0.5 + r*0.5)
            s = self._s.astype(np.float64)
            mono = np.floor(s[:, 0] * 0.5 + s[:, 1] * 0.5).astype(self._s.dtype)
            return AudioSegment(mono[:, None], self.frame_rate)
        raise ValueError("AudioSegment.set_channels only supports mono-to-multi channel and multi-to-mono")

    def set_frame_rate(self, frame_rate: int) -> "AudioSegment":
        if frame_rate == self.frame_rate:
            return self
        raise NotImplementedError("resampling needs pydub/audioop.ratecv (not available in this image)")

    def set_sample_width(self, sample_width: int) -> "AudioSegment":
        if sample_width == self.sample_width:
            return self
        shift = 8 * (sample_width - self.sample_width)
        s = self._s.astype(np.int64)
        s = s << shift if shift > 0 else s >> (-shift)
        return AudioSegment(s.astype(_DTYPES[sample_width]), self.frame_rate)

    # ---- gain
    def apply_gain(self, volume_change: float) -> "AudioSegment":
        factor = db_to_float(float(volume_change))
        info = np.iinfo(self._s.dtype)
        out = np.floor(self._s.astype(np.float64) * factor)
        out = np.clip(out, info.min, info.max).astype(self._s.dtype)
        return AudioSegment(out, self.frame_rate)

    def __add__(self, arg):
        if isinstance(arg, AudioSegment):
            return self.append(arg, crossfade=0)
        return self.apply_gain(arg)

    # ---- slicing / combining (ms)
    def _frames(self, ms: float) -> int:
        return int(ms * self.frame_rate / 1000.0)

    def __getitem__(self, ms) -> "AudioSegment":
        if isinstance(ms, slice):
            start = 0 if ms.start is None else ms.start
            end = len(self) if ms.stop is None else ms.stop
            start = min(max(start + len(self) if start < 0 else start, 0), len(self))
            end = min(max(end + len(self) if end < 0 else end, 0), len(self))
        else:
            start, end = ms, ms + 1
        a, b = self._frames(start), self._frames(end)
        seg = self._s[a:b]
        want = self._frames(end - start)
        if seg.shape[0] < want and want - seg.shape[0] <= self._frames(2):
            seg = np.concatenate([seg, np.zeros((want - seg.shape[0], self.channels), self._s.dtype)])
        return AudioSegment(seg.copy(), self.frame_rate)

    def _sync(self, other: "AudioSegment") -> T.Tuple["AudioSegment", "AudioSegment"]:
        ch = max(self.channels, other.channels)
        if self.frame_rate != other.frame_rate:
            raise NotImplementedError("combining segments of different frame rates needs resampling")
        width = max(self.sample_width, other.sample_width)
        return (self.set_channels(ch).set_sample_width(width), other.set_channels(ch).set_sample_width(width))

    def fade(self, to_gain: float = 0, from_gain: float = 0, start: int = 0, end: T.Optional[int] = None):
        end = len(self) if end is None else end
        a, b = self._frames(start), min(self._frames(end), self._s.shape[0])
        g = np.ones(self._s.shape[0])
        f0, f1 = db_to_float(from_gain), db_to_float(to_gain)
        if b > a:
            g[a:b] = f0 + (f1 - f0) * (np.arange(b - a) / float(b - a))
        g[:a] = f0
        g[b:] = f1
        out = np.floor(self._s.astype(np.float64) * g[:, None])
        info = np.iinfo(self._s.dtype)
        return AudioSegment(np.clip(out, info.min, info.max).astype(self._s.dtype), self.frame_rate)

    def append(self, seg: "AudioSegment", crossfade: int = 100) -> "AudioSegment":
        s1, s2 = self._sync(seg)
        if not crossfade:
            return AudioSegment(np.concatenate([s1._s, s2._s]), s1.frame_rate)
        if crossfade > len(s1) or crossfade > len(s2):
            raise ValueError("Crossfade is longer than a segment")
        n = s1._frames(crossfade)
        head, tail = s1._s[: s1._s.shape[0] - n], s1._s[s1._s.shape[0] - n:]
        ramp = np.arange(n) / float(max(n, 1))
        mix = np.floor(tail.astype(np.float64) * (1 - ramp)[:, None]) + np.floor(
            s2._s[:n].astype(np.float64) * ramp[:, None])
        info = np.iinfo(s1._s.dtype)
        mix = np.clip(mix, info.min, info.max).astype(s1._s.dtype)
        return AudioSegment(np.concatenate([head, mix, s2._s[n:]]), s1.frame_rate)

    def overlay(self, seg: "AudioSegment", position: int = 0) -> "AudioSegment":
        s1, s2 = self._sync(seg)
        out = s1._s.astype(np.int64)
        a = s1._frames(position)
        n = min(s2._s.shape[0], out.shape[0] - a)
        if n > 0:
            out[a : a + n] += s2._s[:n]
        info = np.iinfo(s1._s.dtype)
        return AudioSegment(np.clip(out, info.min, info.max).astype(s1._s.dtype), s1.frame_rate)


def normalize(seg, headroom: float = 0.1):
    """pydub.effects.normalize"""
    peak = seg.max
    if peak == 0:
        return seg
    target_peak = seg.max_possible_amplitude * db_to_float(-headroom)
    return seg.apply_gain(ratio_to_db(target_peak / peak))

"""SpectrogramConverter — H100-native drop-in for riffusion/spectrogram_converter.py.

Same constructor, public attributes (`p`, `device`, `spectrogram_func`,
`inverse_spectrogram_func`, `mel_scaler`, `inverse_mel_scaler`) and methods as the reference
class (spectrogram_converter.py:34-204).  The four transform attributes are callables
Tensor -> Tensor like the torchaudio modules they replace; the two torch-only methods
`mel_amplitudes_from_waveform` / `waveform_from_mel_amplitudes` run fused CUDA kernels
through the C-ABI (include/rf_b200.h).  Nothing here dispatches to torchaudio/cuFFT.
"""
from __future__ import annotations

import math
import threading
import typing as T
import warnings

import numpy as np
import torch

from riffusion import _native
from riffusion.spectrogram_params import SpectrogramParams
from riffusion.util import audio_util, torch_util


def mel_filterbank(
    n_freqs: int, f_min: float, f_max: float, n_mels: int, sample_rate: int,
    norm: T.Optional[str] = None, mel_scale: str = "htk",
) -> torch.Tensor:
    """Triangular mel filterbank (n_freqs, n_mels), float32, on the CPU.

    Restates torchaudio.functional.melscale_fbanks (TA/functional/functional.py:518-587 with
    _hz_to_mel :425-455, _mel_to_hz :458-485, _create_triangular_filterbank :488-513) with the
    same sequence of fp32 torch ops so the matrix is bit-identical to the one the reference's
    MelScale / InverseMelScale modules hold.
    """
    if norm is not None and norm != "slaney":
        raise ValueError('norm must be one of None or "slaney"')
    if mel_scale not in ("slaney", "htk"):
        raise ValueError('mel_scale should be one of "htk" or "slaney".')

    def hz_to_mel(freq: float) -> float:
        if mel_scale == "htk":
            return 2595.0 * math.log10(1.0 + (freq / 700.0))
        f_sp = 200.0 / 3
        mels = freq / f_sp
        min_log_hz = 1000.0
        if freq >= min_log_hz:
            mels = min_log_hz / f_sp + math.log(freq / min_log_hz) / (math.log(6.4) / 27.0)
        return mels

    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    m_pts = torch.linspace(hz_to_mel(f_min), hz_to_mel(f_max), n_mels + 2)
    if mel_scale == "htk":
        f_pts = 700.0 * (10.0 ** (m_pts / 2595.0) - 1.0)
    else:
        f_sp = 200.0 / 3
        f_pts = f_sp * m_pts
        min_log_hz = 1000.0
        min_log_mel = min_log_hz / f_sp
        logstep = math.log(6.4) / 27.0
        log_t = m_pts >= min_log_mel
        f_pts[log_t] = min_log_hz * torch.exp(logstep * (m_pts[log_t] - min_log_mel))

    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    down = (-1.0 * slopes[:, :-2]) / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    fb = torch.max(torch.zeros(1), torch.min(down, up))
    if norm == "slaney":
        fb *= (2.0 / (f_pts[2 : n_mels + 2] - f_pts[:n_mels])).unsqueeze(0)
    if (fb.max(dim=0).values == 0.0).any():
        warnings.warn(
            "At least one mel filterbank has all zero values. "
            f"The value for `n_mels` ({n_mels}) may be set too high. "
            f"Or, the value for `n_freqs` ({n_freqs}) may be set too low."
        )
    return fb


# ------------------------------------------------------------------------------------------
# plan cache (the reference's server rebuilds its converter on every request, server.py:157)
# ------------------------------------------------------------------------------------------
_PLAN_CACHE: T.Dict[T.Tuple, _native.Plan] = {}
_PLAN_LOCK = threading.Lock()


def _device_index(device) -> int:
    if device is None:
        return torch.cuda.current_device() if torch.cuda.is_available() else 0
    d = torch.device(device)
    if d.index is not None:
        return d.index
    return torch.cuda.current_device() if torch.cuda.is_available() else 0


def get_plan(p: SpectrogramParams, full_band: bool, device=None) -> _native.Plan:
    """One plan per (geometry, device): the device tables of a plan are uploaded on first use to the device that is
    current then and stay bound to it (rf_plan checks it), so a second GPU in the same process gets its own plan."""
    key = (_device_index(device), p.sample_rate, p.n_fft, p.win_length, p.hop_length, p.num_frequencies, p.min_frequency,
           p.max_frequency, p.mel_scale_norm, p.mel_scale_type, bool(full_band))
    with _PLAN_LOCK:
        plan = _PLAN_CACHE.get(key)
        if plan is None:
            desc = _native.PlanDesc(
                sample_rate=p.sample_rate, n_fft=p.n_fft, win_length=p.win_length,
                hop_length=p.hop_length, n_mels=p.num_frequencies, f_min=float(p.min_frequency),
                f_max=float(p.max_frequency), mel_norm_slaney=int(p.mel_scale_norm == "slaney"),
                mel_scale_slaney=int(p.mel_scale_type == "slaney"), full_band=int(full_band),
            )
            fb = mel_filterbank(p.n_fft // 2 + 1, float(p.min_frequency), float(p.max_frequency),
                                p.num_frequencies, p.sample_rate, p.mel_scale_norm, p.mel_scale_type)
            window = torch.hann_window(p.win_length)  # periodic, fp32 (TA/_transforms.py:94)
            plan = _native.Plan(desc, window.numpy(), fb.numpy())
            _PLAN_CACHE[key] = plan
    return plan


def _flatten(x: torch.Tensor, keep: int) -> T.Tuple[torch.Tensor, torch.Size]:
    """pack leading dims like torchaudio's `reshape(-1, ...)`"""
    lead = x.shape[: x.dim() - keep]
    return x.reshape((-1,) + tuple(x.shape[x.dim() - keep:])), lead


class _Transform:
    """Callable with the small part of the nn.Module surface callers use."""

    def __init__(self, params: SpectrogramParams, device: str):
        self.p = params
        self.device = torch.device(device)

    def to(self, device) -> "_Transform":
        self.device = torch.device(device)
        return self

    def forward(self, x: torch.Tensor) -> torch.Tensor:  # pragma: no cover - overridden
        raise NotImplementedError

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        return self.forward(x)


class Spectrogram(_Transform):
    """Complex STFT: torchaudio.transforms.Spectrogram(power=None, center=True, reflect)
    as configured at spectrogram_converter.py:47-59."""

    def forward(self, waveform: torch.Tensor) -> torch.Tensor:
        x, lead = _flatten(_native.require_cuda(waveform, "waveform", torch.float32), 1)
        plan = get_plan(self.p, full_band=True, device=x.device)
        B, L = x.shape
        Tn = 1 + L // self.p.hop_length
        spec = torch.empty((B, plan.info.n_freq, Tn), dtype=torch.complex64, device=x.device)
        _native.call("rf_stft", x.device, plan.handle, x.data_ptr(), B, L, spec.data_ptr())
        return spec.reshape(tuple(lead) + spec.shape[-2:])


class MelScale(_Transform):
    """torchaudio.transforms.MelScale as configured at spectrogram_converter.py:75-84."""

    def forward(self, specgram: torch.Tensor) -> torch.Tensor:
        s, lead = _flatten(_native.require_cuda(specgram, "specgram", torch.float32), 2)
        plan = get_plan(self.p, full_band=True, device=s.device)
        B, F, Tn = s.shape
        if F != plan.info.n_freq:
            raise ValueError(f"Expected {plan.info.n_freq} frequency bins. Found: {F}")
        mel = torch.empty((B, self.p.num_frequencies, Tn), dtype=torch.float32, device=s.device)
        _native.call("rf_mel_scale", s.device, plan.handle, s.data_ptr(), B, Tn, mel.data_ptr())
        return mel.reshape(tuple(lead) + mel.shape[-2:])


class InverseMelScale(_Transform):
    """torchaudio.transforms.InverseMelScale (2.x: relu(lstsq(gels))), spectrogram_converter.py:86-99.
    The torchaudio-0.13 SGD variant the reference's kwargs (max_iter, tolerance_*) address is not
    reproducible and not implemented; `max_mel_iters` is accepted and ignored."""

    def forward(self, melspec: torch.Tensor) -> torch.Tensor:
        m, lead = _flatten(_native.require_cuda(melspec, "melspec", torch.float32), 2)
        plan = get_plan(self.p, full_band=False, device=m.device)
        B, n_mels, Tn = m.shape
        if n_mels != self.p.num_frequencies:
            raise ValueError("Expected an input with {} mel bins. Found: {}".format(self.p.num_frequencies, n_mels))
        lin = torch.empty((B, plan.info.n_freq, Tn), dtype=torch.float32, device=m.device)
        _native.call("rf_inverse_mel", m.device, plan.handle, m.data_ptr(), B, Tn, lin.data_ptr())
        return lin.reshape(tuple(lead) + lin.shape[-2:])


class GriffinLim(_Transform):
    """torchaudio.transforms.GriffinLim(power=1, momentum=0.99, rand_init=True, length=None) as
    configured at spectrogram_converter.py:61-73.  Accepts any (.., n_freq, T) magnitudes."""

    momentum = 0.99

    def forward(self, specgram: torch.Tensor, init_angles: T.Optional[torch.Tensor] = None) -> torch.Tensor:
        s, lead = _flatten(_native.require_cuda(specgram, "specgram", torch.float32), 2)
        plan = get_plan(self.p, full_band=True, device=s.device)
        B, F, Tn = s.shape
        if F != plan.info.n_freq:
            raise ValueError(f"Expected {plan.info.n_freq} frequency bins. Found: {F}")
        if init_angles is None:
            # rand_init=True: uniform in the unit square from the global generator
            # (TA/functional/functional.py:309-310)
            init_angles = torch.rand(s.size(), dtype=torch.complex64, device=s.device)
        ang = _native.require_cuda(init_angles, "init_angles", torch.complex64).reshape(B, F, Tn)
        wave = torch.empty((B, self.p.hop_length * (Tn - 1)), dtype=torch.float32, device=s.device)
        nbytes = _native.lib().rf_griffinlim_workspace_bytes(plan.handle, B, Tn)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=s.device)
        _native.call("rf_griffinlim", s.device, plan.handle, s.data_ptr(), ang.data_ptr(), B, Tn,
                     self.p.num_griffin_lim_iters, self.momentum, wave.data_ptr(), ws.data_ptr(), nbytes)
        return wave.reshape(tuple(lead) + wave.shape[-1:])


class SpectrogramConverter:
    """Convert between audio segments and mel-amplitude spectrogram tensors on an H100.

    See the reference class docstring (spectrogram_converter.py:12-32) for the semantics; a
    "spectrogram" here is (channels, n_mels, frames) of mel amplitudes.
    """

    def __init__(self, params: SpectrogramParams, device: str = "cuda"):
        self.p = params
        self.device = torch_util.check_device(device)
        if device.lower().startswith("mps"):
            warnings.warn(
                "WARNING: MPS does not support audio operations, falling back to CPU for them",
                stacklevel=2,
            )
            self.device = "cpu"
        if not str(self.device).lower().startswith("cuda"):
            raise RuntimeError(
                f"SpectrogramConverter(device={device!r}): the H100-native build runs the audio path "
                "in CUDA kernels only; there is no CPU implementation"
            )
        # validates the geometry now (raises NotImplementedError for unsupported sizes)
        get_plan(params, full_band=False, device=self.device)

        self.spectrogram_func = Spectrogram(params, self.device)
        self.inverse_spectrogram_func = GriffinLim(params, self.device)
        self.mel_scaler = MelScale(params, self.device)
        self.inverse_mel_scaler = InverseMelScale(params, self.device)

    # ---- pydub-facing wrappers (spectrogram_converter.py:101-163) --------------------------
    def spectrogram_from_audio(self, audio) -> np.ndarray:
        """AudioSegment -> (channels, n_mels, frames) float32 mel amplitudes."""
        assert int(audio.frame_rate) == self.p.sample_rate, "Audio sample rate must match params"
        waveform = np.array([c.get_array_of_samples() for c in audio.split_to_mono()])
        if waveform.dtype != np.float32:
            waveform = waveform.astype(np.float32)  # raw int16-valued floats, not scaled to [-1, 1]
        waveform_tensor = torch.from_numpy(waveform).to(self.device)
        return self.mel_amplitudes_from_waveform(waveform_tensor).cpu().numpy()

    def audio_from_spectrogram(self, spectrogram: np.ndarray, apply_filters: bool = True):
        """(channels, n_mels, frames) mel amplitudes -> AudioSegment."""
        amplitudes_mel = torch.from_numpy(spectrogram).to(self.device)
        waveform = self.waveform_from_mel_amplitudes(amplitudes_mel)
        segment = audio_util.audio_from_waveform(
            samples=waveform.cpu().numpy(), sample_rate=self.p.sample_rate, normalize=True)
        if apply_filters:
            segment = audio_util.apply_filters(segment, compression=False)
        return segment

    # ---- torch-only core: the C-ABI parity boundary ---------------------------------------
    def mel_amplitudes_from_waveform(self, waveform: torch.Tensor) -> torch.Tensor:
        """(batch, samples) -> (batch, n_mels, frames): STFT, magnitude and mel projection in one
        kernel (spectrogram_converter.py:165-185)."""
        x, lead = _flatten(_native.require_cuda(waveform, "waveform", torch.float32), 1)
        plan = get_plan(self.p, full_band=False, device=x.device)
        B, L = x.shape
        Tn = 1 + L // self.p.hop_length
        mel = torch.empty((B, self.p.num_frequencies, Tn), dtype=torch.float32, device=x.device)
        _native.call("rf_stft_mel", x.device, plan.handle, x.data_ptr(), B, L, mel.data_ptr())
        return mel.reshape(tuple(lead) + mel.shape[-2:])

    def waveform_from_mel_amplitudes(
        self, amplitudes_mel: torch.Tensor, init_angles: T.Optional[torch.Tensor] = None, periodic: bool = False
    ) -> torch.Tensor:
        """(batch, n_mels, frames) -> (batch, hop*(frames-1)): inverse mel + Griffin-Lim, fused
        (spectrogram_converter.py:187-204).  `init_angles` (batch, n_freq, frames) complex64
        overrides the random phase initialisation (used by the parity tests).

        `periodic` (seamless loops) -> (batch, hop*frames): the waveform is one period of a looping signal; frame t is
        centred at sample t*hop and every sample index wraps around, so the end runs into the start without a seam
        (include/rf_b200.h: rf_mel_to_wave_periodic)."""
        m, lead = _flatten(_native.require_cuda(amplitudes_mel, "amplitudes_mel", torch.float32), 2)
        plan = get_plan(self.p, full_band=False, device=m.device)
        B, n_mels, Tn = m.shape
        if n_mels != self.p.num_frequencies:
            raise ValueError("Expected an input with {} mel bins. Found: {}".format(self.p.num_frequencies, n_mels))
        F = plan.info.n_freq
        if init_angles is None:
            init_angles = torch.rand((B, F, Tn), dtype=torch.complex64, device=m.device)
        ang = _native.require_cuda(init_angles, "init_angles", torch.complex64).reshape(B, F, Tn)
        if periodic:
            wave = torch.empty((B, self.p.hop_length * Tn), dtype=torch.float32, device=m.device)
            nbytes = _native.lib().rf_mel_to_wave_periodic_workspace_bytes(plan.handle, B, Tn)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=m.device)
            _native.call("rf_mel_to_wave_periodic", m.device, plan.handle, m.data_ptr(), ang.data_ptr(), B, Tn,
                         self.p.num_griffin_lim_iters, GriffinLim.momentum, wave.data_ptr(), ws.data_ptr(), nbytes)
            return wave.reshape(tuple(lead) + wave.shape[-1:])
        wave = torch.empty((B, self.p.hop_length * (Tn - 1)), dtype=torch.float32, device=m.device)
        nbytes = _native.lib().rf_griffinlim_workspace_bytes(plan.handle, B, Tn)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=m.device)
        _native.call("rf_mel_to_wave", m.device, plan.handle, m.data_ptr(), ang.data_ptr(), B, Tn,
                     self.p.num_griffin_lim_iters, GriffinLim.momentum, wave.data_ptr(), ws.data_ptr(), nbytes)
        return wave.reshape(tuple(lead) + wave.shape[-1:])

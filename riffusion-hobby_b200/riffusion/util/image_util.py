"""Spectrogram <-> image quantisation (reference: riffusion/util/image_util.py).

Host (numpy/PIL) versions with the reference's exact semantics, plus device-side equivalents
(`spectrogram_from_image_device`, `image_from_spectrogram_device`) that run the same arithmetic in
CUDA kernels so amplitudes never leave the GPU between the converter stages.
"""
from __future__ import annotations

import typing as T

import numpy as np
import torch
from PIL import Image

from riffusion.spectrogram_params import SpectrogramParams


def image_from_spectrogram(spectrogram: np.ndarray, power: float = 0.25) -> Image.Image:
    """(channels, frequency, time) amplitudes -> PIL image (frequency, time, RGB).

    image_util.py:13-56: divide by the max over ALL channels, apply the power curve, scale to 255,
    invert, truncate to uint8; one channel is replicated to RGB, two channels go to (0, ch0, ch1);
    finally the frequency axis is flipped so low frequencies are at the bottom.
    """
    peak = np.max(spectrogram)
    scaled = np.power(spectrogram / peak, power) * 255
    pixels = (255 - scaled).astype(np.uint8)

    n_ch = pixels.shape[0]
    if n_ch == 1:
        image = Image.fromarray(pixels[0], mode="L").convert("RGB")
    elif n_ch == 2:
        rgb = np.stack([np.zeros_like(pixels[0]), pixels[0], pixels[1]], axis=-1)
        image = Image.fromarray(rgb, mode="RGB")
    else:
        raise NotImplementedError(f"Unsupported number of channels: {n_ch}")
    return image.transpose(Image.Transpose.FLIP_TOP_BOTTOM)


def _rgb_array(image: Image.Image) -> np.ndarray:
    if image.mode in ("P", "L"):
        image = image.convert("RGB")
    return np.array(image)


def spectrogram_from_image(
    image: Image.Image, power: float = 0.25, stereo: bool = False, max_value: float = 30e6
) -> np.ndarray:
    """PIL image -> (channels, frequency, time) float32 amplitudes (image_util.py:59-110).

    Mono reads the R plane only, stereo reads G and B; values are ((255 - u8)/255)^(1/power) *
    max_value with the frequency axis flipped back.
    """
    planes = _rgb_array(image.transpose(Image.Transpose.FLIP_TOP_BOTTOM)).transpose(2, 0, 1)
    planes = planes[[1, 2]] if stereo else planes[0:1]
    data = planes.astype(np.float32)
    data = 255 - data
    data = data / 255
    data = np.power(data, 1 / power)
    return data * max_value


def exif_from_image(pil_image: Image.Image) -> T.Dict[str, T.Any]:
    """EXIF of a spectrogram image as {tag name: value} (image_util.py:113-122)."""
    exif = pil_image.getexif()
    if exif is None or len(exif) == 0:
        return {}
    return {SpectrogramParams.ExifTags(key).name: val for key, val in exif.items()}


# ------------------------------------------------------------------------------ device versions
def spectrogram_from_image_device(
    image: T.Union[Image.Image, torch.Tensor], power: float = 0.25, stereo: bool = False,
    max_value: float = 30e6, device: str = "cuda",
) -> torch.Tensor:
    """Same arithmetic as `spectrogram_from_image`, on the GPU: uint8 (H, W, 3) in, float32
    (channels, H, W) out — 1 byte read and 4 written per pixel, no host float array."""
    from riffusion import _native

    if isinstance(image, Image.Image):
        rgb = torch.from_numpy(_rgb_array(image)).to(device)
    else:
        rgb = image
    rgb = _native.require_cuda(rgb, "image", torch.uint8)
    H, W, _ = _native.operand(rgb, "image", torch.uint8, shape=(_native.ANY, _native.ANY, 3)).shape
    out = torch.empty((2 if stereo else 1, H, W), dtype=torch.float32, device=rgb.device)
    _native.call("rf_image_to_mel", rgb.device, rgb.data_ptr(), H, W, int(stereo), float(power), float(max_value),
                 out.data_ptr())
    return out


def image_from_spectrogram_device(spectrogram: torch.Tensor, power: float = 0.25) -> T.Tuple[torch.Tensor, torch.Tensor]:
    """Same arithmetic as `image_from_spectrogram`, on the GPU. Returns (uint8 (H, W, 3) tensor,
    0-dim float32 tensor holding the max over all channels = EXIF MAX_VALUE)."""
    from riffusion import _native

    s = _native.require_cuda(spectrogram, "spectrogram", torch.float32)
    C, H, W = _native.operand(s, "spectrogram", torch.float32, shape=(_native.ANY,) * 3).shape
    if C not in (1, 2):
        raise NotImplementedError(f"Unsupported number of channels: {C}")
    img = torch.empty((H, W, 3), dtype=torch.uint8, device=s.device)
    mx = torch.empty((), dtype=torch.float32, device=s.device)
    _native.call("rf_mel_to_image", s.device, s.data_ptr(), C, H, W, float(power), img.data_ptr(), mx.data_ptr())
    return img, mx

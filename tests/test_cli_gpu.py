"""CLI end to end on the GPU, mirroring the reference's CLI tests on its own fixture (test/audio_to_image_test.py,
test/image_to_audio_test.py, test/spectrogram_image_converter_test.py): clip_2 WAV -> PNG -> WAV."""
import numpy as np
import pytest
from PIL import Image

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("stereo", [False, True])
def test_audio_to_image_then_image_to_audio(native_lib, golden, tmp_path, stereo):
    from scipy.io import wavfile

    from riffusion import cli
    from riffusion.spectrogram_params import SpectrogramParams
    from riffusion.util.audio_util import AudioSegment

    g = golden["clip2"]
    wavfile.write(tmp_path / "clip.wav", int(g["rate"]), g["wav"])
    args = ["audio-to-image", "--audio", str(tmp_path / "clip.wav"), "--image", str(tmp_path / "clip.png")]
    cli.main(args + (["--stereo"] if stereo else []))
    img = Image.open(tmp_path / "clip.png")
    assert img.mode == "RGB" and img.width == round(5678 / 10) and img.height == 512      # audio_to_image_test.py:73-75
    arr = np.array(img)
    if stereo:
        assert np.all(arr[:, :, 0] == 0)                                                  # :81-83
        diff = np.abs(arr.astype(np.int16) - g["stereo_png"].astype(np.int16))
        assert diff.max() <= 1 and (diff != 0).mean() < 1e-3                              # the reference's own fixture image
    else:
        assert np.array_equal(arr[:, :, 0], arr[:, :, 1]) and np.array_equal(arr[:, :, 0], arr[:, :, 2])   # :84-87
    params = SpectrogramParams.from_exif(img.getexif())
    assert params == SpectrogramParams(stereo=stereo)                                     # :89-99
    cli.main(["image-to-audio", "--image", str(tmp_path / "clip.png"), "--audio", str(tmp_path / "out.wav")])
    seg = AudioSegment.from_file(str(tmp_path / "out.wav"))
    assert seg.frame_rate == 44100                                                        # image_to_audio_test.py:55
    assert abs(seg.duration_seconds * 1000 - 5678) < 12                                   # :58-60 (10 ms + 1 hop)
    assert seg.channels == (2 if stereo else 1) and seg.sample_width == 2                 # :63-67


def test_server_compute_request_on_gpu(native_lib, tmp_path):
    """riffusion/server.py:116-183 end to end on the GPU: riffuse (reduced-width UNet + full VAE + library's CLIP encoder) ->
    SpectrogramImageConverter.audio_from_spectrogram_image -> JSON with a base64 JPEG and base64 audio of 5.11 s"""
    import base64
    import io
    import json
    import sys
    from pathlib import Path

    import numpy as np
    import torch
    from PIL import Image

    sys.path.insert(0, str(Path(__file__).parent / "golden"))
    from prompt_stub import StubTokenizer
    from riffusion import sd15_spec, server
    from riffusion.clip_b200 import ClipTextB200
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.unet_b200 import UNetB200
    from riffusion.vae_b200 import VaeB200

    c = (64, 128, 128, 128)
    unet = UNetB200(sd15_spec.random_state_dict(sd15_spec.unet_spec(c, cross_attention_dim=768), 0), device="cuda",
                    block_out_channels=c, heads=4)
    vae = VaeB200(sd15_spec.random_state_dict(sd15_spec.vae_spec(), 1), device="cuda")
    pipe = RiffusionPipeline(vae=vae, unet=unet, text_encoder=ClipTextB200.random_init(seed=2, layers=2), tokenizer=StubTokenizer(),
                             device="cuda")
    rgb = np.load(Path(__file__).parent / "golden" / "og_beat.npz")["rgb"]
    Image.fromarray(rgb, mode="RGB").save(tmp_path / "og_beat.png")
    payload = {"alpha": 0.5, "num_inference_steps": 10, "seed_image_id": "og_beat",
               "start": {"prompt": "church bells on sunday", "seed": 42}, "end": {"prompt": "jazz with (piano:1.3)", "seed": 123}}
    out = json.loads(server.run_inference(payload, pipe, tmp_path))
    assert abs(out["duration_s"] - 5.11) < 0.01
    img = Image.open(io.BytesIO(base64.decodebytes(out["image"].split(",", 1)[1].encode())))
    assert img.size == (512, 512)
    assert len(base64.decodebytes(out["audio"].split(",", 1)[1].encode())) > 2 * 225351
    torch.cuda.synchronize()

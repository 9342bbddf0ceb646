"""(f)-3: ClipTextB200 (the CLIP text encoder on the wgmma GEMM / causal-attention kernels) against the reference's own
dependency for this module — `transformers.CLIPTextModel` (what diffusers loads as `pipe.text_encoder`,
riffusion/riffusion_pipeline.py:92-102,177-191) — built offline with the CLIP-L/14 text configuration and random-init
weights; both sides hold the same fp16-representable parameters.  The oracle here is PINNED: it is the real library."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.fixture(scope="module")
def clip_pair(native_lib):
    from transformers import CLIPTextConfig, CLIPTextModel

    from riffusion.clip_b200 import ClipTextB200

    torch.manual_seed(0)
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                         num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu")
    ref = CLIPTextModel(cfg).eval()
    with torch.no_grad():
        for n, p in ref.named_parameters():
            if p.dim() == 1 and "norm" in n and n.endswith("weight"):
                p.copy_(1.0 + 0.1 * torch.randn_like(p))          # exercise the affine paths
            elif p.dim() == 1:
                p.copy_(0.05 * torch.randn_like(p))
            p.copy_(p.half().float())
    return ref.cuda(), ClipTextB200(ref.state_dict(), device="cuda")


@torch.no_grad()
def test_clip_text_encoder_matches_transformers(clip_pair):
    ref, ours = clip_pair
    torch.manual_seed(1)
    ids = torch.randint(0, 49406, (3, 77))
    ids[:, 0] = 49406
    ids[0, 9:] = 49407                                   # BOS, 8 tokens, EOS padding — what the tokenizer produces
    ids[1, 40:] = 49407
    want = ref(ids.cuda())[0]
    got = ours(ids)[0]
    assert got.shape == (3, 77, 768) and got.dtype == torch.float16 and torch.isfinite(got).all()
    want16 = ref.half()(ids.cuda())[0].float()
    ref.float()
    e, e16 = rel_l2(got, want), rel_l2(want16, want)
    print(f"CLIP text encoder: ours vs transformers fp32 {e:.3e}; transformers fp16 vs fp32 {e16:.3e}")
    assert e <= 1.25 * e16 + 2e-4 and e < 3e-3
    # causality: a change of token j must not alter the outputs at positions < j
    ids2 = ids.clone()
    ids2[:, 30] = (ids2[:, 30] + 17) % 49000
    got2 = ours(ids2)[0]
    assert torch.equal(got2[:, :30], got[:, :30]) and not torch.equal(got2[:, 30:], got[:, 30:])


@torch.no_grad()
def test_pipeline_embeds_text_through_b200_encoder(clip_pair):
    """embed_text / embed_text_weighted (riffusion_pipeline.py:177-206) with the library's encoder behind the tokenizer seam"""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).parent / "golden"))
    from prompt_stub import StubTokenizer
    from riffusion.riffusion_pipeline import RiffusionPipeline

    ref, ours = clip_pair
    tok = StubTokenizer()
    pipe = RiffusionPipeline(vae=None, unet=None, text_encoder=ours, tokenizer=tok, device="cuda")
    e = pipe.embed_text("church bells on sunday")
    ids = tok("church bells on sunday", padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
    assert e.shape == (1, 77, 768) and rel_l2(e, ref(ids.cuda())[0]) < 3e-3
    w = pipe.embed_text_weighted("church (bells:1.3) on sunday")
    assert w.shape == (1, 77, 768) and rel_l2(w, e) > 1e-3
    assert abs(float(w.float().mean()) - float(e.float().mean())) < 1e-3

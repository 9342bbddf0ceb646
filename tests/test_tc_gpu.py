"""GPU numerics of the wgmma GEMM / implicit-GEMM convolution against plain PyTorch fp32 references
of the same op (fp16-rounded inputs, fp32 math).  Tolerance: fp16 output rounding (2^-11 relative) plus
fp32 accumulation-order noise: |err| <= 2e-3 * max|ref| everywhere."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _close(got, ref, tol=2e-3):
    err = (got.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= tol * scale, f"max err {err:.4e} vs scale {scale:.4e}"


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 320, 320), (4096, 1280, 320), (77, 640, 768), (130, 40, 4096),
                                   (2, 1280, 320)])
def test_gemm_matches_torch(native_lib, M, N, K):
    from riffusion import tc_ops

    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device="cuda") * 0.5).half()
    b = (torch.randn(N, K, device="cuda") * 0.5).half()
    bias = torch.randn(N, device="cuda").half()
    res = torch.randn(M, N, device="cuda").half()
    ref = a.float() @ b.float().t()
    _close(tc_ops.gemm(a, b).reshape(M, N), ref)
    _close(tc_ops.gemm(a, b, bias=bias, residual=res, alpha=0.5).reshape(M, N), 0.5 * ref + bias.float() + res.float())
    ref_silu = torch.nn.functional.silu(ref + bias.float())
    _close(tc_ops.gemm(a, b, bias=bias, act=tc_ops.ACT_SILU).reshape(M, N), ref_silu)
    f32 = tc_ops.gemm(a, b, out_dtype=torch.float32).reshape(M, N)
    assert f32.dtype == torch.float32
    _close(f32, ref, tol=2e-5)


@pytest.mark.parametrize("M,C", [(300, 320), (4096, 640), (77, 1280)])
def test_gemm_geglu_epilogue(native_lib, M, C):
    """ff.net.0.proj + GEGLU fused (diffusers GEGLU: hidden, gate = proj(x).chunk(2); hidden * gelu(gate))"""
    import torch.nn.functional as F

    from riffusion import tc_ops as ops

    torch.manual_seed(M + C)
    x = torch.randn(M, C, device="cuda").half()
    w = (torch.randn(8 * C, C, device="cuda") / C ** 0.5).half()
    b = (0.1 * torch.randn(8 * C, device="cuda")).half()
    h, gate = (x.float() @ w.float().t() + b.float()).chunk(2, dim=-1)
    ref = h * F.gelu(gate)
    got = ops.gemm(x, ops.interleave_geglu(w), bias=ops.interleave_geglu(b), act=ops.ACT_GEGLU)
    assert got.shape[-2:] == (M, 4 * C)
    assert (got.float().reshape(M, 4 * C) - ref).abs().max() < 2e-2
    unfused = ops.geglu(ops.gemm(x, w, bias=b).reshape(M, 8 * C))
    assert (got.float().reshape(M, 4 * C) - unfused.float()).abs().max() < 1e-2


def test_gemm_batched_strided_heads(native_lib):
    """attention-shaped operands: Q/K views (B, heads, tokens, d) of a (B, tokens, heads*d) tensor, d = 40
    (K tail zero-filled by TMA), per-row bias, fp32 and fp16 outputs"""
    from riffusion import tc_ops

    torch.manual_seed(0)
    B, Hh, Tq, Tk, d = 2, 8, 192, 77, 40
    q = (torch.randn(B, Tq, Hh * d, device="cuda") * 0.3).half()
    k = (torch.randn(B, Tk, Hh * d, device="cuda") * 0.3).half()
    qv = q.view(B, Tq, Hh, d).permute(0, 2, 1, 3)
    kv = k.view(B, Tk, Hh, d).permute(0, 2, 1, 3)
    s = tc_ops.gemm(qv, kv, alpha=d ** -0.5)
    ref = torch.einsum("bhqd,bhkd->bhqk", qv.float(), kv.float()) * d ** -0.5
    assert s.shape == (B, Hh, Tq, Tk)
    _close(s, ref)
    # V^T produced directly by swapping operand roles: (heads*d, tokens) = W (Cout, Cin) . X (tokens, Cin)^T
    x = (torch.randn(B, Tk, 768, device="cuda") * 0.3).half()
    w = (torch.randn(Hh * d, 768, device="cuda") * 0.05).half()
    bias = torch.randn(Hh * d, device="cuda").half()
    vt = torch.empty(B, 1, Hh * d, 80, dtype=torch.float16, device="cuda")[..., :Tk]     # pitch 80 (16-byte rows)
    tc_ops.gemm(w, x.unsqueeze(1), bias=bias, bias_per_row=True, out=vt)
    ref_vt = torch.einsum("ck,btk->bct", w.float(), x.float()) + bias.float()[None, :, None]
    _close(vt.reshape(B, Hh * d, Tk), ref_vt)


@pytest.mark.parametrize("B,H,W,C1,C2,Cout,k,stride", [
    (2, 64, 64, 320, 0, 320, 3, 1), (2, 32, 32, 640, 0, 640, 3, 1), (2, 16, 16, 1280, 1280, 1280, 3, 1),
    (2, 8, 8, 1280, 0, 1280, 3, 1), (3, 8, 8, 1280, 0, 1280, 3, 1), (2, 64, 64, 320, 0, 320, 3, 2),
    (2, 16, 16, 640, 0, 640, 3, 2), (2, 32, 32, 960, 0, 640, 1, 1), (1, 128, 128, 256, 0, 128, 3, 1),
    (2, 32, 32, 320, 640, 64, 3, 1), (2, 16, 16, 1280, 640, 1280, 1, 1),
])
def test_conv_matches_torch(native_lib, B, H, W, C1, C2, Cout, k, stride):
    from riffusion import tc_ops

    torch.manual_seed(H + C1 + Cout + k)
    x = (torch.randn(B, H, W, C1, device="cuda") * 0.5).half()
    x2 = (torch.randn(B, H, W, C2, device="cuda") * 0.5).half() if C2 else None
    w = (torch.randn(Cout, C1 + C2, k, k, device="cuda") * (C1 + C2) ** -0.5 / k).half()
    bias = torch.randn(Cout, device="cuda").half()
    temb = torch.randn(B, Cout, device="cuda").half()
    xin = x if x2 is None else torch.cat([x, x2], dim=3)
    ref = torch.nn.functional.conv2d(xin.permute(0, 3, 1, 2).float(), w.float(), bias.float(), stride=stride,
                                     padding=1 if k == 3 else 0)
    ref = (ref + temb.float()[:, :, None, None]).permute(0, 2, 3, 1)
    wp = tc_ops.pack_conv_weight(w)
    got = tc_ops.conv2d(x, wp, x2=x2, bias=bias, bias_per_image=temb, stride=stride)
    assert got.shape == ref.shape
    _close(got, ref)
    res = torch.randn_like(got)
    got2 = tc_ops.conv2d(x, wp, x2=x2, bias=bias, residual=res, stride=stride)
    _close(got2, ref - temb.float()[:, None, None, :] + res.float())


@pytest.mark.parametrize("B,heads,Nq,Nk,d", [(2, 8, 4096, 4096, 40), (2, 8, 1024, 1024, 80), (2, 8, 256, 256, 160),
                                             (3, 8, 64, 64, 160), (2, 8, 4096, 77, 40), (1, 8, 1024, 77, 80),
                                             (2, 8, 256, 77, 160), (1, 4, 200, 300, 16), (1, 2, 128, 129, 64)])
def test_fused_attention_matches_torch(native_lib, B, heads, Nq, Nk, d):
    """fused QK^T -> softmax -> PV (wgmma) vs fp32 torch attention on the same fp16 inputs;
    UNet self-/cross-attention shapes plus ragged sizes (query / key tails, single and odd tile counts)"""
    from riffusion import tc_ops

    torch.manual_seed(Nq + Nk + d)
    C = heads * d
    q = (torch.randn(B, Nq, C, device="cuda") * 1.5).half()
    k = (torch.randn(B, Nk, C, device="cuda") * 1.5).half()
    v = torch.randn(B, Nk, C, device="cuda").half()
    pitch = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, C, pitch, dtype=torch.float16, device="cuda")
    vt[..., :Nk] = v.transpose(1, 2)
    qh, kh, vh = (t.float().view(B, -1, heads, d).transpose(1, 2) for t in (q, k, v))
    ref = torch.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, dim=-1) @ vh
    ref = ref.transpose(1, 2).reshape(B, Nq, C)
    got = tc_ops.attention(q, k, vt, heads, Nk)
    assert got.shape == ref.shape and torch.isfinite(got).all()
    _close(got, ref, tol=4e-3)
    assert float((got.float() - ref).norm() / ref.norm()) < 2e-3


@pytest.mark.parametrize("Nk,d", [(1024, 40), (700, 40), (512, 80), (384, 64), (300, 96)])
def test_fused_attention_growing_scores(native_lib, Nk, d):
    """online softmax: the keys are ordered so that the row maximum keeps growing along the key axis (forces the
    rescale of the running accumulators on every key tile) with peaked softmax rows (large logits)"""
    from riffusion import tc_ops

    torch.manual_seed(Nk + d)
    B, heads, Nq = 1, 2, 200
    C = heads * d
    a = 0.5 + torch.rand(B, Nq, 1, device="cuda")
    q = (a + 0.5 * torch.randn(B, Nq, C, device="cuda")).half()            # q_i ~ a_i * ones + noise
    ramp = torch.linspace(0.0, 6.0, Nk, device="cuda")[None, :, None]
    k = (ramp + 0.5 * torch.randn(B, Nk, C, device="cuda")).half()          # logits ~ a_i * ramp_j * sqrt(d)
    v = torch.randn(B, Nk, C, device="cuda").half()
    pitch = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, C, pitch, dtype=torch.float16, device="cuda")
    vt[..., :Nk] = v.transpose(1, 2)
    qh, kh, vh = (t.float().view(B, -1, heads, d).transpose(1, 2) for t in (q, k, v))
    logits = qh @ kh.transpose(-1, -2) * d ** -0.5
    assert float(logits.max() - logits.min()) > 30          # the test is only meaningful with a wide logit range
    ref = (torch.softmax(logits, dim=-1) @ vh).transpose(1, 2).reshape(B, Nq, C)
    got = tc_ops.attention(q, k, vt, heads, Nk)
    assert torch.isfinite(got).all()
    _close(got, ref, tol=6e-3)
    assert float((got.float() - ref).norm() / ref.norm()) < 3e-3


# ----------------------------------------------------------------------------------------------- tile widths
def _tile_env(bn, bres="1"):
    import os

    if bn is None:
        os.environ.pop("RF_GEMM_BN", None)
    else:
        os.environ["RF_GEMM_BN"] = str(bn)
    if bres == "0":
        os.environ["RF_GEMM_BRES"] = "0"
    else:
        os.environ.pop("RF_GEMM_BRES", None)


@pytest.mark.parametrize("bres", ["1", "0"])
@pytest.mark.parametrize("bn", [None, 64, 128, 160])
def test_large_gemm_matches_torch_every_tile_width(native_lib, bn, bres):
    """problems of many waves with every output-tile width (RF_GEMM_BN) and with the B-stationary mode on and off, ragged M
    (a partial last 128-row block), bias / SiLU / residual / GEGLU epilogues, batched operands; results also compared with
    the default tile choice"""
    import torch.nn.functional as F

    from riffusion import tc_ops as ops

    try:
        for (M, N, K) in ((128 * 297 - 58, 320, 320), (40000, 1280, 640), (36000, 640, 320), (38000, 256, 192)):
            if bn == 160 and N % 160:
                continue
            torch.manual_seed(M + N)
            a = (torch.randn(M, K, device="cuda") * 0.5).half()
            b = (torch.randn(N, K, device="cuda") * 0.5).half()
            bias = torch.randn(N, device="cuda").half()
            res = torch.randn(M, N, device="cuda").half()
            ref = a.float() @ b.float().t()
            _tile_env(bn, bres)
            g1 = ops.gemm(a, b).reshape(M, N)
            g2 = ops.gemm(a, b, bias=bias, residual=res, alpha=0.5).reshape(M, N)
            g3 = ops.gemm(a, b, bias=bias, act=ops.ACT_SILU).reshape(M, N)
            _close(g1, ref)
            _close(g2, 0.5 * ref + bias.float() + res.float())
            _close(g3, F.silu(ref + bias.float()))
            _tile_env(None)
            s1 = ops.gemm(a, b).reshape(M, N)
            # same K order and fp32 accumulation for every tile width: at most isolated fp16 rounding flips
            assert float((g1 != s1).float().mean()) < 1e-3 and float((g1.float() - s1.float()).abs().max()) <= 2e-3 * float(ref.abs().max()), (M, N, K)
        # GEGLU epilogue (N = 8C interleaved) and a batched V^T-style product with 3 row blocks per batch entry
        _tile_env(bn, bres)
        M, C = 33000, 320
        x = torch.randn(M, C, device="cuda").half()
        w = (torch.randn(8 * C, C, device="cuda") / C ** 0.5).half()
        bb = (0.1 * torch.randn(8 * C, device="cuda")).half()
        h, gate = (x.float() @ w.float().t() + bb.float()).chunk(2, dim=-1)
        got = ops.gemm(x, ops.interleave_geglu(w), bias=ops.interleave_geglu(bb), act=ops.ACT_GEGLU).reshape(M, 4 * C)
        assert (got.float() - h * F.gelu(gate)).abs().max() < 2e-2
        Bt, T = 24, 4096
        xt = (torch.randn(Bt, T, 320, device="cuda") * 0.3).half()
        wv = (torch.randn(320, 320, device="cuda") * 0.05).half()
        vt = torch.empty(Bt, 1, 320, T, dtype=torch.float16, device="cuda")
        ops.gemm(wv, xt.unsqueeze(1), out=vt)
        _close(vt.reshape(Bt, 320, T), torch.einsum("ck,btk->bct", wv.float(), xt.float()))
    finally:
        _tile_env(None)


@pytest.mark.parametrize("B,H,W,C1,C2,Cout,k,stride", [
    (8, 64, 64, 320, 0, 320, 3, 1), (16, 32, 32, 640, 0, 640, 3, 1), (16, 32, 32, 640, 640, 1280, 3, 1),
    (16, 64, 64, 320, 0, 320, 3, 2), (13, 48, 48, 128, 0, 256, 3, 1), (24, 32, 32, 960, 0, 640, 1, 1),
    (3, 256, 256, 128, 0, 128, 3, 1),
])
def test_large_conv_matches_torch_every_tile_width(native_lib, B, H, W, C1, C2, Cout, k, stride):
    """implicit-GEMM convolution at batch sizes of many waves: each CTA gathers its 128 output pixels (TMA im2col boxes),
    stride 2, channel concat through the second tensor map, per-image bias, residual; vs torch with the default tile
    width, and the default vs the 128- and 64-column tiles"""
    from riffusion import tc_ops

    torch.manual_seed(H + C1 + Cout + k)
    x = (torch.randn(B, H, W, C1, device="cuda") * 0.5).half()
    x2 = (torch.randn(B, H, W, C2, device="cuda") * 0.5).half() if C2 else None
    w = (torch.randn(Cout, C1 + C2, k, k, device="cuda") * (C1 + C2) ** -0.5 / k).half()
    bias = torch.randn(Cout, device="cuda").half()
    temb = torch.randn(B, Cout, device="cuda").half()
    xin = x if x2 is None else torch.cat([x, x2], dim=3)
    ref = torch.nn.functional.conv2d(xin.permute(0, 3, 1, 2).float(), w.float(), bias.float(), stride=stride,
                                     padding=1 if k == 3 else 0)
    ref = (ref + temb.float()[:, :, None, None]).permute(0, 2, 3, 1)
    wp = tc_ops.pack_conv_weight(w)
    try:
        _tile_env(None)
        got = tc_ops.conv2d(x, wp, x2=x2, bias=bias, bias_per_image=temb, stride=stride)
        _close(got, ref)
        res = torch.randn_like(got)
        got2 = tc_ops.conv2d(x, wp, x2=x2, bias=bias, residual=res, stride=stride)
        _close(got2, ref - temb.float()[:, None, None, :] + res.float())
        for bn in (128, 64):
            _tile_env(bn)
            other = tc_ops.conv2d(x, wp, x2=x2, bias=bias, bias_per_image=temb, stride=stride)
            assert float((got != other).float().mean()) < 1e-3, bn
    finally:
        _tile_env(None)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 16, 16, 1280, 1280), (2, 32, 32, 640, 640), (1, 8, 8, 128, 64),
                                            (16, 32, 32, 640, 640), (3, 64, 64, 256, 256), (2, 5, 7, 64, 192)])
def test_fused_upsample_conv_matches_torch(native_lib, B, H, W, Cin, Cout):
    """Upsample2D = F.interpolate(nearest, 2x) + conv 3x3 pad 1, computed as four 2x2 sub-pixel convolutions on the
    low-resolution input (rf_conv2d_f16 pad_mode 2): vs torch on the upsampled tensor, and vs the unfused kernels"""
    import torch.nn.functional as F

    from riffusion import tc_ops as ops

    torch.manual_seed(H + Cin + Cout)
    x = (torch.randn(B, H, W, Cin, device="cuda") * 0.5).half()
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda") * Cin ** -0.5 / 3).half()
    bias = torch.randn(Cout, device="cuda").half()
    ref = F.conv2d(F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest"), w.float(), bias.float(),
                   padding=1).permute(0, 2, 3, 1)
    got = ops.conv2d_upsample2x(x, ops.pack_upsample_weight(w), bias=bias)
    assert got.shape == (B, 2 * H, 2 * W, Cout)
    _close(got, ref, tol=3e-3)             # + one fp16 rounding of the pre-summed phase weights
    unfused = ops.conv2d(ops.upsample2x(x), ops.pack_conv_weight(w), bias=bias)
    assert float((got.float() - unfused.float()).norm() / unfused.float().norm()) < 1e-3


def test_b_stationary_gemm_matches_torch_and_streaming_kernel(native_lib):
    """K <= 320, N = 320 / 480 problems with many row blocks run B-stationary (the CTA keeps its weight tile in shared
    memory and streams only A): GEMM with bias / residual / SiLU, ragged M, K = 192 (3 slabs), and a 1x1 convolution;
    vs torch and vs the streaming kernel (RF_GEMM_BRES=0)"""
    import os

    import torch.nn.functional as F

    from riffusion import tc_ops as ops

    try:
        for (M, N, K) in ((128 * 300 + 77, 320, 320), (45000, 480, 192), (128 * 296, 320, 256)):
            torch.manual_seed(M + N + K)
            a = (torch.randn(M, K, device="cuda") * 0.5).half()
            b = (torch.randn(N, K, device="cuda") * 0.5).half()
            bias = torch.randn(N, device="cuda").half()
            res = torch.randn(M, N, device="cuda").half()
            ref = a.float() @ b.float().t()
            os.environ.pop("RF_GEMM_BRES", None)
            g1 = ops.gemm(a, b, bias=bias, residual=res).reshape(M, N)
            g2 = ops.gemm(a, b, bias=bias, act=ops.ACT_SILU).reshape(M, N)
            _close(g1, ref + bias.float() + res.float())
            _close(g2, F.silu(ref + bias.float()))
            os.environ["RF_GEMM_BRES"] = "0"
            s1 = ops.gemm(a, b, bias=bias, residual=res).reshape(M, N)
            assert torch.equal(g1, s1), (M, N, K)            # same slab order, same accumulation
        os.environ.pop("RF_GEMM_BRES", None)
        x = (torch.randn(10, 64, 64, 320, device="cuda") * 0.5).half()
        w = (torch.randn(320, 320, 1, 1, device="cuda") * 320 ** -0.5).half()
        bias = torch.randn(320, device="cuda").half()
        ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias.float()).permute(0, 2, 3, 1)
        got = ops.conv2d(x, ops.pack_conv_weight(w), bias=bias)
        _close(got, ref)
    finally:
        os.environ.pop("RF_GEMM_BRES", None)

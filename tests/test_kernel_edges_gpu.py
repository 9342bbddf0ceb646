"""Kernel-level edge cases of path (b) against fp64 torch references computed from the same fp16 inputs.

Every check is elementwise:  |got - ref64| <= ulp16(ref64) + (arithmetic term), where ulp16(r) is the spacing of fp16
numbers at |r| (2^-24 in the subnormal range), i.e. one fp16 rounding of the output with a factor 2 of headroom, and
the arithmetic term is the fp32 error of the kernel's own evaluation, stated per test:
  * GEMM / convolution: fp32 accumulation, <= 2^-15 * sum_k |a_k b_k| (x 1.2 through an activation, whose slope is
    below 1.2);
  * GroupNorm / LayerNorm: the fp32 statistics and the affine form x * (rstd gamma) + (beta - mean rstd gamma),
    <= 2^-20 * ((|x| + |mean|) * rstd * |gamma| + |beta|)  (rstd from fp32 sums: about 2^-20 relative);
  * attention: P is rounded to fp16 before P V and the row sum, <= 2^-10 * max|V| of the (image, head).
The shapes, strides, alignments and values are the ones where the kernels change path: split-K and its second stage,
the scalar epilogue fall-backs, tiny / ragged images, template head dims, the causal mask, offsets with mean >> std.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ulp16(r: torch.Tensor) -> torch.Tensor:
    e = torch.floor(torch.log2(r.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _check(got, ref, extra=0.0, what=""):
    """got: kernel output; ref: fp64 reference; extra: fp64 tensor / float, the arithmetic error term"""
    ref = ref.double()
    err = (got.double() - ref).abs()
    tol = _ulp16(ref) + extra
    bad = ~(err <= tol)
    if bad.any():
        ratio = (err / tol).nan_to_num(float("inf"))
        i = int(ratio.flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} outside the bound; worst: got "
                             f"{got.double().flatten()[i].item():.6g}, ref {ref.flatten()[i].item():.6g}, err "
                             f"{err.flatten()[i].item():.3e}, tol {tol.flatten()[i].item() if torch.is_tensor(tol) else tol:.3e}")


def _all_fp16() -> torch.Tensor:
    """the 63,488 finite fp16 values (both zeros, subnormals, +-65504)"""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    v = bits.view(torch.float16)
    return v[torch.isfinite(v)].to(DEV)


# ============================================================================================ GroupNorm / LayerNorm
def _norm_tol(x64, mean, rstd, gamma, beta):
    return 2.0 ** -20 * ((x64.abs() + mean.abs()) * rstd * gamma.abs() + beta.abs())


def _silu_tol(pre64, tol_pre):
    """SiLU on the GroupNorm output: silu(v) = h + h tanh(h), h = v/2, with tanh.approx.f32 (relative error about 2^-11,
    taken as 2^-10), after an input error tol_pre (slope of silu < 1.1)"""
    h = 0.5 * pre64
    return 1.1 * tol_pre + 2.0 ** -10 * (h * torch.tanh(h)).abs()


def _gn_case(B, H, W, C, G, offset, std, eps, silu, x2_channels=0, const_group=None, seed=0):
    from riffusion import tc_ops as ops

    torch.manual_seed(seed)
    C1 = C - x2_channels
    xf = offset + std * torch.randn(B, H, W, C, device=DEV)
    if const_group is not None:
        cpg = C // G
        xf[1 % B, ..., const_group * cpg:(const_group + 1) * cpg] = offset + 3.0 * std
    x = xf.half()
    gamma = (1 + 0.2 * torch.randn(C, device=DEV)).half()
    beta = (0.2 * torch.randn(C, device=DEV)).half()
    if x2_channels:
        a, c = x[..., :C1].contiguous(), x[..., C1:].contiguous()
        got = ops.group_norm(a, gamma, beta, G, eps, silu, x2=c)
    else:
        got = ops.group_norm(x, gamma, beta, G, eps, silu)
    x64 = x.double()
    xg = x64.reshape(B, H * W, G, C // G)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(xg.var(dim=(1, 3), unbiased=False, keepdim=True) + eps)
    mean = mean.expand_as(xg).reshape(B, H, W, C)
    rstd = rstd.expand_as(xg).reshape(B, H, W, C)
    pre = F.group_norm(x64.permute(0, 3, 1, 2), G, gamma.double(), beta.double(), eps=eps).permute(0, 2, 3, 1)
    tol = _norm_tol(x64, mean, rstd, gamma.double(), beta.double())
    what = f"GroupNorm B{B} {H}x{W} C{C} G{G} offset {offset} std {std} eps {eps} silu {silu} x2 {x2_channels}"
    if silu:
        _check(got, F.silu(pre), _silu_tol(pre, tol), what)
    else:
        _check(got, pre, tol, what)
    return got


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("offset,std", [(0.0, 1.0), (64.0, 1.0), (256.0, 1.0), (8.0, 0.01)])
def test_group_norm_offset_statistics(native_lib, offset, std, silu):
    """mean >> std: the variance must not come from E[x^2] - mean^2 in fp32; C = 320, G = 32 (10 channels per group: a
    thread's 8-channel octet straddles two groups), HW = 1024, plus the two-source (channel concatenation) form with a
    group across the seam (C = 640 + 320, 30 channels per group)"""
    _gn_case(2, 32, 32, 320, 32, offset, std, 1e-5, silu)
    _gn_case(2, 16, 16, 960, 32, offset, std, 1e-5, silu, x2_channels=320)


@pytest.mark.parametrize("B,H,W,C,G,offset,std,eps", [
    (16, 64, 64, 320, 32, 64.0, 1.0, 1e-5),      # slab 64
    (16, 63, 63, 320, 32, 8.0, 0.01, 1e-6),      # slab 64, HW not a multiple of the slab
    (8, 256, 256, 128, 32, 64.0, 1.0, 1e-5),     # slab 256, 4 channels per group
    (4, 1, 1, 320, 32, 0.0, 1.0, 1e-5),          # HW = 1: 10 elements per group
    (3, 7, 9, 640, 32, 256.0, 1.0, 1e-6),        # HW = 63: a partial slab of 32
    (2, 5, 7, 2560, 32, 8.0, 0.01, 1e-5),        # widest supported row
])
def test_group_norm_slabs_and_sizes(native_lib, B, H, W, C, G, offset, std, eps):
    for silu in (False, True):
        _gn_case(B, H, W, C, G, offset, std, eps, silu)


def test_group_norm_constant_group_and_determinism(native_lib):
    """a constant group has variance 0: its outputs are beta (GroupNorm) and silu(beta) (with SiLU); repeated runs are
    bit-identical, and the two-source form equals the same call on the concatenated tensor bit for bit"""
    from riffusion import tc_ops as ops

    for silu in (False, True):
        got = _gn_case(2, 16, 16, 320, 32, 64.0, 1.0, 1e-5, silu, const_group=5)
        got2 = _gn_case(2, 16, 16, 320, 32, 64.0, 1.0, 1e-5, silu, const_group=5)
        assert torch.equal(got, got2)
    torch.manual_seed(3)
    a = (100 + torch.randn(2, 8, 8, 640, device=DEV)).half()
    c = (100 + torch.randn(2, 8, 8, 320, device=DEV)).half()
    g = torch.randn(960, device=DEV).half()
    b = torch.randn(960, device=DEV).half()
    assert torch.equal(ops.group_norm(a, g, b, 32, 1e-5, True, x2=c),
                       ops.group_norm(torch.cat([a, c], dim=-1), g, b, 32, 1e-5, True))


def test_group_norm_rejects_too_many_groups_before_launch(native_lib):
    """more than 64 groups is unsupported; the call is refused before the first kernel is launched"""
    from riffusion import tc_ops as ops

    x = torch.randn(1, 4, 4, 256, device=DEV).half()
    g = torch.ones(256, device=DEV).half()
    with pytest.raises(NotImplementedError, match="at most 64 groups"):
        ops.group_norm(x, g, g, 128, 1e-5, False)
    torch.cuda.synchronize()


def _ln_case(rows, C, offset, std, eps, unaligned=False, const_row=False, seed=0):
    from riffusion import tc_ops as ops

    torch.manual_seed(seed)
    xf = offset + std * torch.randn(rows, C, device=DEV)
    if const_row:
        xf[rows // 2] = offset + 2.0 * std
    if unaligned:      # a row pitch of C at a 2-element (4-byte) offset: not 16-byte aligned -> the generic kernel
        buf = torch.empty(rows * C + 2, dtype=torch.float16, device=DEV)
        x = buf[2:].view(rows, C)
        x.copy_(xf.half())
    else:
        x = xf.half()
    gamma = (1 + 0.2 * torch.randn(C, device=DEV)).half()
    beta = (0.2 * torch.randn(C, device=DEV)).half()
    got = ops.layer_norm(x, gamma, beta, eps)
    x64 = x.double()
    mean = x64.mean(dim=1, keepdim=True)
    rstd = 1.0 / torch.sqrt(x64.var(dim=1, unbiased=False, keepdim=True) + eps)
    ref = F.layer_norm(x64, (C,), gamma.double(), beta.double(), eps=eps)
    _check(got, ref, _norm_tol(x64, mean, rstd, gamma.double(), beta.double()),
           f"LayerNorm rows {rows} C {C} offset {offset} std {std} eps {eps} unaligned {unaligned}")


@pytest.mark.parametrize("C,unaligned", [(320, False), (640, False), (1280, False), (96, False), (320, True)])
@pytest.mark.parametrize("offset,std", [(0.0, 1.0), (64.0, 1.0), (128.0, 1.0), (4.0, 0.01)])
def test_layer_norm_offset_statistics(native_lib, C, unaligned, offset, std):
    """vectorised widths 320 / 640 / 1280 and the generic kernel (C = 96, or 320 at an unaligned address); 1001 rows
    (a partial last block), one constant row, eps 1e-5 and 1e-6"""
    _ln_case(1001, C, offset, std, 1e-5, unaligned, const_row=True)
    _ln_case(77, C, offset, std, 1e-6, unaligned)


# ============================================================================================ GEMM epilogues
def _gemm_ref(a, b, bias=None, bias_per_row=False, residual=None, alpha=1.0, act=0):
    from riffusion import tc_ops as ops

    acc = alpha * (a.double() @ b.double().transpose(-1, -2))
    s = abs(alpha) * (a.double().abs() @ b.double().abs().transpose(-1, -2))
    if bias is not None:
        acc = acc + (bias.double()[:, None] if bias_per_row else bias.double())
    if act == ops.ACT_SILU:
        acc = F.silu(acc)
    elif act == ops.ACT_QUICK_GELU:
        acc = acc * torch.sigmoid(1.702 * acc)
    if residual is not None:
        acc = acc + residual.double()
    return acc, (1.2 if act else 1.0) * 2.0 ** -15 * s


class _WsSpy:
    """wraps tc_ops._workspace: records the split-K scratch requests; `withhold` runs the un-split kernel instead"""

    def __init__(self, monkeypatch, withhold=False):
        from riffusion import tc_ops

        self.requests, self.withhold = [], withhold
        self._orig = getattr(tc_ops._workspace, "_orig", tc_ops._workspace)     # not an earlier spy
        monkeypatch.setattr(tc_ops, "_workspace", self)

    def __call__(self, nbytes, desc, device):
        self.requests.append(int(nbytes))
        return None if self.withhold else self._orig(nbytes, desc, device)


@pytest.mark.parametrize("M,N,K", [(77, 768, 3072), (130, 40, 4096), (1, 768, 3072), (64, 320, 2048)])
def test_gemm_split_k_epilogues_match_unsplit(native_lib, monkeypatch, M, N, K):
    """small-M problems with a long K take split-K (fp32 partials + k_splitk_reduce); the same problem with the workspace
    withheld runs the un-split kernel.  Both vs fp64 and vs each other (same operands, different fp32 order: within
    two accumulation bounds and one fp16 ulp), for every epilogue the reduce stage implements"""
    from riffusion import tc_ops as ops

    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).half()
    b = (torch.randn(N, K, device=DEV) * K ** -0.5).half()
    col = torch.randn(N, device=DEV).half()
    row = torch.randn(M, device=DEV).half()
    res = torch.randn(M, N, device=DEV).half()
    cases = [
        dict(bias=col, residual=res, alpha=0.5),
        dict(bias=row, bias_per_row=True, act=ops.ACT_SILU),
        dict(bias=col, act=ops.ACT_QUICK_GELU, alpha=1.5),
        dict(bias=row, bias_per_row=True, residual=res, act=ops.ACT_QUICK_GELU),
        dict(act=ops.ACT_SILU, residual=res),
        dict(bias=col, out_dtype=torch.float32),
    ]
    for kw in cases:
        out_dtype = kw.pop("out_dtype", torch.float16)
        ref, acc_tol = _gemm_ref(a, b, **kw)
        outs = []
        for withhold in (False, True):
            spy = _WsSpy(monkeypatch, withhold)
            got = ops.gemm(a, b, out_dtype=out_dtype, **kw).reshape(M, N)
            assert spy.requests and spy.requests[-1] > 0, f"split-K was not taken for {(M, N, K)}"
            if out_dtype == torch.float32:
                err = (got.double() - ref).abs()
                assert bool((err <= acc_tol + 2.0 ** -22 * ref.abs()).all()), (kw, float(err.max()))
            else:
                _check(got, ref, acc_tol, f"gemm {(M, N, K)} {kw} split={not withhold}")
            outs.append(got)
        if out_dtype == torch.float32:
            assert bool(((outs[0].double() - outs[1].double()).abs() <= 2 * acc_tol).all())
        else:
            _check(outs[0], outs[1].double(), 2 * acc_tol, f"split vs un-split {(M, N, K)} {kw}")


@pytest.mark.parametrize("N", [1, 8, 33, 77])
@pytest.mark.parametrize("M,K", [(1, 77), (77, 64), (130, 77), (300, 136)])
def test_gemm_scalar_epilogue_paths(native_lib, M, N, K):
    """out, residual and column bias as slices at a 4-element (8-byte) offset of wider tensors: not 16-byte aligned, so
    the epilogue takes its scalar loads / stores; N below one 32-column run or ragged; K with a tail (operands with a
    row pitch of K rounded up to 8, the tail zero-filled by TMA); M = 1.  Plus the aligned variants of the same call"""
    from riffusion import tc_ops as ops

    torch.manual_seed(M * 100 + N + K)
    pk = (K + 7) // 8 * 8
    a = (torch.randn(M, pk, device=DEV) * 0.5).half()[:, :K]
    b = (torch.randn(N, pk, device=DEV) * K ** -0.5).half()[:, :K]
    wide_bias = torch.randn(N + 8, device=DEV).half()
    wide_res = torch.randn(M, N + 8, device=DEV).half()
    for off in (4, 0):
        bias, res = wide_bias[off:off + N], wide_res[:, off:off + N]
        for act in (ops.ACT_NONE, ops.ACT_SILU, ops.ACT_QUICK_GELU):
            out_wide = torch.full((M, N + 8), float("nan"), dtype=torch.float16, device=DEV)
            out = out_wide[:, off:off + N]
            ops.gemm(a, b, bias=bias, residual=res, alpha=0.75, act=act, out=out)
            ref, acc_tol = _gemm_ref(a, b, bias=bias, residual=res, alpha=0.75, act=act)
            _check(out, ref, acc_tol, f"gemm {(M, N, K)} offset {off} act {act}")
            # nothing outside the view was written
            assert torch.isnan(out_wide[:, :off]).all() and torch.isnan(out_wide[:, off + N:]).all()
        got = ops.gemm(a, b, bias=bias, out_dtype=torch.float32).reshape(M, N)
        ref, acc_tol = _gemm_ref(a, b, bias=bias)
        assert bool(((got.double() - ref).abs() <= acc_tol + 2.0 ** -22 * ref.abs()).all()), (M, N, K, off)


def test_gemm_row_bias_unaligned(native_lib):
    """per-row bias at an odd element offset (read one element per row in the epilogue)"""
    from riffusion import tc_ops as ops

    torch.manual_seed(5)
    M, N, K = 333, 96, 128
    a = torch.randn(M, K, device=DEV).half()
    b = (torch.randn(N, K, device=DEV) * K ** -0.5).half()
    bias = torch.randn(M + 1, device=DEV).half()[1:]
    ref, acc_tol = _gemm_ref(a, b, bias=bias, bias_per_row=True, act=ops.ACT_SILU)
    _check(ops.gemm(a, b, bias=bias, bias_per_row=True, act=ops.ACT_SILU).reshape(M, N), ref, acc_tol, "row bias")


@pytest.mark.parametrize("bcast", ["a", "b"])
def test_gemm_broadcast_operand(native_lib, bcast):
    """one operand shared by the whole batch (batch stride 0), two batch dims"""
    from riffusion import tc_ops as ops

    torch.manual_seed(7)
    M, N, K = 150, 72, 200
    a = (torch.randn(1 if bcast == "a" else 3, 1 if bcast == "a" else 2, M, K, device=DEV) * 0.5).half()
    b = (torch.randn(1 if bcast == "b" else 3, 1 if bcast == "b" else 2, N, K, device=DEV) * K ** -0.5).half()
    bias = torch.randn(N, device=DEV).half()
    got = ops.gemm(a, b, bias=bias, alpha=0.3)
    assert got.shape == (3, 2, M, N)
    ref, acc_tol = _gemm_ref(a.expand(3, 2, M, K), b.expand(3, 2, N, K), bias=bias, alpha=0.3)
    _check(got, ref, acc_tol, f"broadcast {bcast}")


# ============================================================================================ exhaustive activations
def test_activation_epilogues_on_every_fp16_value(native_lib):
    """all 63,488 finite fp16 values v, each within one fp16 ulp of fp64:
    GEMM epilogue SiLU / quick_gelu with zero operands and the values as per-row bias (out[m, :] = act(v[m]));
    GEGLU epilogue (gelu_erf_fast): a one-hot A column carries v into the gate rows, the value rows get bias 1;
    rf_silu_f16 and rf_geglu_f16 on the same values"""
    from riffusion import tc_ops as ops

    v = _all_fp16()
    M = v.numel()
    v64 = v.double()
    zeros_a = torch.zeros(M, 64, dtype=torch.float16, device=DEV)
    zeros_b = torch.zeros(8, 64, dtype=torch.float16, device=DEV)
    silu64 = F.silu(v64)
    qgelu64 = v64 * torch.sigmoid(1.702 * v64)
    gelu64 = F.gelu(v64)            # exact erf form
    for act, ref in ((ops.ACT_SILU, silu64), (ops.ACT_QUICK_GELU, qgelu64)):
        got = ops.gemm(zeros_a, zeros_b, bias=v, bias_per_row=True, act=act).reshape(M, 8)
        _check(got, ref[:, None].expand(M, 8), 0.0, f"gemm epilogue act {act}")
    inner = 16
    a = torch.zeros(M, 64, dtype=torch.float16, device=DEV)
    a[:, 0] = v
    w = torch.zeros(2 * inner, 64, dtype=torch.float16, device=DEV)
    w[inner:, 0] = 1.0                                  # gate rows pick column 0
    bias = torch.cat([torch.ones(inner), torch.zeros(inner)]).half().to(DEV)     # value rows: 0 + 1
    got = ops.gemm(a, ops.interleave_geglu(w), bias=ops.interleave_geglu(bias), act=ops.ACT_GEGLU).reshape(M, inner)
    _check(got, gelu64[:, None].expand(M, inner), 0.0, "GEGLU epilogue gelu_erf_fast")
    _check(ops.silu(v), silu64, 0.0, "rf_silu_f16")
    x = torch.stack([torch.ones_like(v), torch.ones_like(v), v, v], dim=1).contiguous()
    _check(ops.geglu(x), gelu64[:, None].expand(M, 2), 0.0, "rf_geglu_f16")


# ============================================================================================ convolution
def _conv_ref(x, w, bias, stride, padding, bias_per_image=None, act=0, x2=None, residual=None, far_pad=False):
    xin = x if x2 is None else torch.cat([x, x2], dim=3)
    x64 = xin.permute(0, 3, 1, 2).double()
    if far_pad:
        x64 = F.pad(x64, (0, 1, 0, 1))
    ref = F.conv2d(x64, w.double(), None if bias is None else bias.double(), stride=stride, padding=padding)
    s = F.conv2d(x64.abs(), w.double().abs(), None, stride=stride, padding=padding)
    ref, s = ref.permute(0, 2, 3, 1), s.permute(0, 2, 3, 1)
    if bias_per_image is not None:
        ref = ref + bias_per_image.double()[:, None, None, :]
    if act == 1:
        ref = F.silu(ref)
    if residual is not None:
        ref = ref + residual.double()
    return ref, (1.2 if act else 1.0) * 2.0 ** -15 * s


@pytest.mark.parametrize("H,W", [(1, 1), (2, 3), (3, 5), (7, 9), (1, 130), (130, 3)])
def test_conv_tiny_and_ragged_images(native_lib, H, W):
    """tile shapes chosen from the output size (bw / bh / bb: a tile of 128 single pixels of 128 images, partial tiles
    past W = 128, W = 3 with 2-pixel tile rows), stride 1 and 2, kernel 1 and 3, a Cout of 96 (a partial column tile);
    per-image bias and a SiLU epilogue"""
    from riffusion import tc_ops as ops

    torch.manual_seed(H * 1000 + W)
    B, C, Cout = 3, 64, 96
    x = (torch.randn(B, H, W, C, device=DEV) * 0.5).half()
    temb = torch.randn(B, Cout, device=DEV).half()
    bias = torch.randn(Cout, device=DEV).half()
    for k in (1, 3):
        w = (torch.randn(Cout, C, k, k, device=DEV) * (C * k * k) ** -0.5).half()
        wp = ops.pack_conv_weight(w)
        for stride in (1, 2):
            for act in (ops.ACT_NONE, ops.ACT_SILU):
                got = ops.conv2d(x, wp, bias=bias, bias_per_image=temb, stride=stride, act=act)
                ref, tol = _conv_ref(x, w, bias, stride, 1 if k == 3 else 0, bias_per_image=temb, act=act)
                assert got.shape == ref.shape, (got.shape, ref.shape)
                _check(got, ref, tol, f"conv {H}x{W} k{k} s{stride} act {act}")


@pytest.mark.parametrize("H,W", [(2, 3), (7, 9), (8, 8), (130, 3), (3, 130)])
def test_conv_far_edge_padding(native_lib, H, W):
    """pad_mode 1 (VAE Downsample2D): F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 convolution without padding;
    with a residual"""
    from riffusion import tc_ops as ops

    torch.manual_seed(H + W)
    B, C, Cout = 2, 128, 128
    x = (torch.randn(B, H, W, C, device=DEV) * 0.5).half()
    w = (torch.randn(Cout, C, 3, 3, device=DEV) * (9 * C) ** -0.5).half()
    bias = torch.randn(Cout, device=DEV).half()
    ref, tol = _conv_ref(x, w, bias, 2, 0, far_pad=True)
    got = ops.conv2d(x, ops.pack_conv_weight(w), bias=bias, stride=2, pad_far_edge_only=True)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    _check(got, ref, tol, f"far-edge pad {H}x{W}")
    res = torch.randn(got.shape, device=DEV).half()
    got = ops.conv2d(x, ops.pack_conv_weight(w), bias=bias, stride=2, pad_far_edge_only=True, residual=res)
    _check(got, ref + res.double(), tol, f"far-edge pad {H}x{W} + residual")


@pytest.mark.parametrize("H,W", [(7, 9), (16, 16)])
def test_conv_concat_stride2(native_lib, H, W):
    """channel concatenation through the second tensor map, at stride 2 (1x1 and 3x3)"""
    from riffusion import tc_ops as ops

    torch.manual_seed(H * W)
    B, C1, C2, Cout = 2, 64, 128, 64
    x = (torch.randn(B, H, W, C1, device=DEV) * 0.5).half()
    x2 = (torch.randn(B, H, W, C2, device=DEV) * 0.5).half()
    for k in (1, 3):
        w = (torch.randn(Cout, C1 + C2, k, k, device=DEV) * ((C1 + C2) * k * k) ** -0.5).half()
        got = ops.conv2d(x, ops.pack_conv_weight(w), x2=x2, stride=2, act=ops.ACT_SILU)
        ref, tol = _conv_ref(x, w, None, 2, 1 if k == 3 else 0, x2=x2, act=1)
        _check(got, ref, tol, f"concat conv {H}x{W} k{k}")


@pytest.mark.parametrize("offset", [4, 64])
def test_conv_bias_per_image_column_slice(native_lib, offset):
    """the time-embedding bias as a column slice of a wider (B, n) matrix (row pitch n): at a 4-element offset the rows
    are not 16-byte aligned and the epilogue reads them one element at a time"""
    from riffusion import tc_ops as ops

    torch.manual_seed(offset)
    B, H, W, C, Cout = 3, 12, 12, 128, 128
    x = (torch.randn(B, H, W, C, device=DEV) * 0.5).half()
    w = (torch.randn(Cout, C, 3, 3, device=DEV) * (9 * C) ** -0.5).half()
    wide = torch.randn(B, 3 * Cout, device=DEV).half()
    temb = wide[:, offset:offset + Cout]
    res = torch.randn(B, H, W, Cout, device=DEV).half()
    got = ops.conv2d(x, ops.pack_conv_weight(w), bias_per_image=temb, residual=res)
    ref, tol = _conv_ref(x, w, None, 1, 1, bias_per_image=temb, residual=res)
    _check(got, ref, tol, f"bias_per_image offset {offset}")


def test_conv_split_k_matches_unsplit(native_lib, monkeypatch):
    """a 2 x 8 x 8 x 1280 -> 1280 3x3 convolution has one row of tiles and 180 K slabs: split-K, with the per-image
    bias, residual and SiLU applied by the second stage; vs fp64 and vs the same call with the workspace withheld"""
    from riffusion import tc_ops as ops

    torch.manual_seed(11)
    B, H, W, C, Cout = 2, 8, 8, 1280, 1280
    x = (torch.randn(B, H, W, C, device=DEV) * 0.5).half()
    w = (torch.randn(Cout, C, 3, 3, device=DEV) * (9 * C) ** -0.5).half()
    wp = ops.pack_conv_weight(w)
    bias = torch.randn(Cout, device=DEV).half()
    temb = torch.randn(B, 2 * Cout, device=DEV).half()[:, Cout:]
    res = torch.randn(B, H, W, Cout, device=DEV).half()
    for kw, act in ((dict(bias=bias, bias_per_image=temb), ops.ACT_NONE), (dict(bias=bias, residual=res), ops.ACT_SILU)):
        ref, tol = _conv_ref(x, w, bias, 1, 1, bias_per_image=kw.get("bias_per_image"), act=act,
                             residual=kw.get("residual"))
        outs = []
        for withhold in (False, True):
            spy = _WsSpy(monkeypatch, withhold)
            got = ops.conv2d(x, wp, act=act, **kw)
            assert spy.requests and spy.requests[-1] > 0, "split-K was not taken"
            _check(got, ref, tol, f"conv split-K withheld={withhold} act {act}")
            outs.append(got)
        _check(outs[0], outs[1].double(), 2 * tol, "conv split vs un-split")


# ============================================================================================ attention
def _attn_ref(q, k, v, heads, causal=False):
    B, Nq, C = q.shape
    Nk, d = k.shape[1], C // heads
    qh, kh, vh = (t.double().view(B, -1, heads, d).transpose(1, 2) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) * d ** -0.5
    if causal:
        mask = torch.arange(Nk, device=DEV)[None, :] > torch.arange(Nq, device=DEV)[:, None]
        s = s.masked_fill(mask, float("-inf"))
    o = torch.softmax(s, dim=-1) @ vh
    vmax = vh.abs().amax(dim=(2, 3), keepdim=True)           # per (image, head)
    tol = (2.0 ** -10 * vmax).expand_as(o)
    return o.transpose(1, 2).reshape(B, Nq, C), tol.transpose(1, 2).reshape(B, Nq, C)


def _run_attn(q, k, v, heads, causal=False, pad=16):
    from riffusion import tc_ops as ops

    B, Nk, C = k.shape
    pitch = (Nk + 7) // 8 * 8 + pad
    vt = torch.full((B, C, pitch), float("nan"), dtype=torch.float16, device=DEV)     # [Nk, pitch) must never be read
    vt[..., :Nk] = v.transpose(1, 2)
    return ops.attention(q, k, vt, heads, Nk, causal=causal)


@pytest.mark.parametrize("d", [8, 24, 48, 56, 64, 72, 104, 112, 120, 128, 136, 176, 192])
def test_attention_head_dims(native_lib, d):
    """every head-dim template (NV = 48 .. 192, DPAD 64 / 128 / 192) and padded NV widths; B = 3, 5 heads with different
    scales per head, 130 queries (a partial query block), 100 keys (a partial key tile), NaN in the V^T pitch columns;
    rows 0-3 of every image are uniform (q = 0) and rows 4-7 one-hot (q = 4 k_j)"""
    torch.manual_seed(d)
    B, heads, Nq, Nk = 3, 5, 130, 100
    C = heads * d
    hs = torch.linspace(0.5, 2.0, heads, device=DEV).repeat_interleave(d)
    q = torch.randn(B, Nq, C, device=DEV) * hs
    k = torch.randn(B, Nk, C, device=DEV)
    v = torch.randn(B, Nk, C, device=DEV) * hs
    q[:, :4] = 0
    for r, j in enumerate((0, 37, 63, 99)):
        q[:, 4 + r] = 4 * k[:, j]
    q, k, v = q.half(), k.half(), v.half()
    got = _run_attn(q, k, v, heads)
    assert torch.isfinite(got).all()
    ref, tol = _attn_ref(q, k, v, heads)
    _check(got, ref, tol, f"attention d {d}")


@pytest.mark.parametrize("Nq,Nk", [(1, 1), (7, 7), (64, 64), (65, 65), (77, 77), (128, 128), (100, 77), (40, 77),
                                   (200, 128), (77, 3)])
def test_attention_causal(native_lib, Nq, Nk):
    """causal mask (key j visible to query i iff j <= i), square and Nq != Nk, d = 64 and 40; NaN V^T padding"""
    for d in (64, 40):
        torch.manual_seed(Nq * 7 + Nk + d)
        B, heads = 3, 5
        q = (torch.randn(B, Nq, heads * d, device=DEV) * 1.5).half()
        k = (torch.randn(B, Nk, heads * d, device=DEV) * 1.5).half()
        v = torch.randn(B, Nk, heads * d, device=DEV).half()
        got = _run_attn(q, k, v, heads, causal=True)
        assert torch.isfinite(got).all()
        ref, tol = _attn_ref(q, k, v, heads, causal=True)
        _check(got, ref, tol, f"causal attention Nq {Nq} Nk {Nk} d {d}")


@pytest.mark.parametrize("Nk,d,causal", [(129, 64, True), (77, 120, True), (77, 200, False)])
def test_attention_rejects_unsupported(native_lib, Nk, d, causal):
    """rejected on the host before any launch (RF_ERR_UNSUPPORTED): causal with Nk > 128 or d > 112, and d > 192"""
    from riffusion import tc_ops as ops

    heads, B, Nq = 2, 1, 16
    q = torch.zeros(B, Nq, heads * d, dtype=torch.float16, device=DEV)
    k = torch.zeros(B, Nk, heads * d, dtype=torch.float16, device=DEV)
    vt = torch.zeros(B, heads * d, (Nk + 7) // 8 * 8, dtype=torch.float16, device=DEV)
    with pytest.raises(NotImplementedError, match="causal mask is implemented" if causal else "head dim > 192"):
        ops.attention(q, k, vt, heads, Nk, causal=causal)
    torch.cuda.synchronize()


# ============================================================================================ element-wise
def test_guided_eps_bit_identical_to_torch(native_lib):
    """cfg_pndm_step's guided eps reproduces torch's fp16 CUDA expression eu + g * (et - eu) bit for bit"""
    from riffusion import tc_ops as ops

    torch.manual_seed(0)
    B = 3
    eps_pair = (torch.randn(2 * B, 4, 64, 64, device=DEV) * torch.tensor([1.0, 30.0, 0.01, 300.0], device=DEV)[:, None, None]).half()
    sample = torch.randn(B, 4, 64, 64, device=DEV).half()
    eu, et = eps_pair[:B], eps_pair[B:]
    for g in (7.5, 1.0, 0.3, 12.345):
        eps, _ = ops.cfg_pndm_step(eps_pair, g, [], (1.0, 0.0, 0.0, 0.0), sample, 0.9, 0.1)
        assert torch.equal(eps, eu + g * (et - eu)), g
        assert torch.equal(eps.view(torch.int16), (eu + g * (et - eu)).view(torch.int16)), g


@pytest.mark.parametrize("n_hist", [0, 1, 2, 3])
def test_cfg_pndm_step_history_and_no_eps(native_lib, n_hist):
    """prev = ca * x - cb * (c0 eps + c1 h1 + c2 h2 + c3 h3) with 0-3 history tensors, vs fp64 (fp32 arithmetic:
    <= 2^-21 * (|ca x| + |cb| sum |c_j h_j|)); want_eps=False gives the same prev bit for bit"""
    from riffusion import tc_ops as ops

    torch.manual_seed(n_hist)
    B = 2
    eps_pair = torch.randn(2 * B, 4, 32, 32, device=DEV).half()
    sample = (torch.randn(B, 4, 32, 32, device=DEV) * 3).half()
    hist = [torch.randn(B, 4, 32, 32, device=DEV).half() for _ in range(n_hist)]
    coef = (55 / 24, -59 / 24, 37 / 24, -9 / 24)[:n_hist + 1] + (0.0,) * (3 - n_hist)
    ca, cb, g = 1.02, 0.13, 7.5
    eps, prev = ops.cfg_pndm_step(eps_pair, g, hist, coef, sample, ca, cb)
    none, prev2 = ops.cfg_pndm_step(eps_pair, g, hist, coef, sample, ca, cb, want_eps=False)
    assert none is None and torch.equal(prev, prev2)
    eu, et = eps_pair[:B], eps_pair[B:]
    e0 = eu + g * (et - eu)
    assert torch.equal(eps, e0)
    terms = [e0] + hist
    e = sum(c * t.double() for c, t in zip(coef, terms))
    ref = ca * sample.double() - cb * e
    mag = abs(ca) * sample.double().abs() + abs(cb) * sum(abs(c) * t.double().abs() for c, t in zip(coef, terms))
    _check(prev, ref, 2.0 ** -21 * mag, f"cfg_pndm_step {n_hist} history tensors")


def test_axpby_mask_blend(native_lib):
    """scheduler add_noise with an inpainting mask: y = (a x + b n) m + z (1 - m).  m = 1 equals the call without a mask
    bit for bit, m = 0 returns z bit for bit, a random mask is within fp32 arithmetic + one fp16 rounding"""
    from riffusion import tc_ops as ops

    torch.manual_seed(2)
    shape = (2, 4, 64, 65)
    x, nz, z = (torch.randn(shape, device=DEV).half() for _ in range(3))
    a, b = 0.8, 0.6
    plain = ops.axpby(x, nz, a, b)
    _check(plain, a * x.double() + b * nz.double(), 2.0 ** -22 * (a * x.double().abs() + b * nz.double().abs()), "axpby")
    ones, zeros = torch.ones_like(x), torch.zeros_like(x)
    assert torch.equal(ops.axpby(x, nz, a, b, mask=ones, z=z).view(torch.int16), plain.view(torch.int16))
    assert torch.equal(ops.axpby(x, nz, a, b, mask=zeros, z=z), z)
    m = torch.rand(shape, device=DEV).half()
    got = ops.axpby(x, nz, a, b, mask=m, z=z)
    v = a * x.double() + b * nz.double()
    ref = v * m.double() + z.double() * (1 - m.double())
    mag = (a * x.double().abs() + b * nz.double().abs()) * m.double() + z.double().abs()
    _check(got, ref, 2.0 ** -21 * mag, "axpby with mask")


@pytest.mark.parametrize("n", [1, 31, 32, 33, 77, 1000, 4096])
def test_softmax_rows_widths_and_extreme_logits(native_lib, n):
    """one warp per row over n of `pitch` = n + 9 columns (odd pitch: no vector access assumed), the padding zeroed;
    rows of moderate logits, rows near +6e4 and near -6e4 (fp16 spacing 32 there: ties share the mass exactly), and a
    constant row.  exp and the normalisation in fp32: <= 2^-19 relative on top of one fp16 rounding"""
    from riffusion import tc_ops as ops

    torch.manual_seed(n)
    rows, pitch = 24, n + 9
    x = torch.randn(rows, pitch, device=DEV) * 3
    x[8:12] = 6.0e4 + 200 * torch.randn(4, pitch, device=DEV)
    x[12:16] = -6.0e4 + 200 * torch.randn(4, pitch, device=DEV)
    x[16] = 5.0
    x = x.clamp(-65504, 65504).half()
    ref = torch.softmax(x[:, :n].double(), dim=-1)
    got = ops.softmax_rows_(x.clone(), n)
    assert bool((got[:, n:] == 0).all())
    _check(got[:, :n], ref, 2.0 ** -19 * ref, f"softmax_rows n {n}")

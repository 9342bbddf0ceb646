"""k_tc_gemm epilogue branches at many work units per CTA, against fp64 torch references from the same fp16 inputs.

The consumer warps hand each finished tile to the epilogue warps through the staging tile and go on to the next unit,
so every branch is run here on problems where each persistent CTA walks several units (the handoff passes through
many phases and the epilogue warps recompute each unit's coordinates): per-row bias + SiLU, column bias + quick_gelu,
fp32 output with a residual, and split-K partial stores with more units than SMs.  The bound is the one of
test_kernel_edges_gpu.py: one fp16 rounding of the output plus the fp32 accumulation term 2^-15 * sum_k |a_k b_k|
(x 1.2 through an activation).
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ref(a, b, bias=None, bias_per_row=False, residual=None, alpha=1.0, act=0):
    from riffusion import tc_ops as ops

    acc = alpha * (a.double() @ b.double().t())
    s = abs(alpha) * (a.double().abs() @ b.double().abs().t())
    if bias is not None:
        acc = acc + (bias.double()[:, None] if bias_per_row else bias.double())
    if act == ops.ACT_SILU:
        acc = F.silu(acc)
    elif act == ops.ACT_QUICK_GELU:
        acc = acc * torch.sigmoid(1.702 * acc)
    if residual is not None:
        acc = acc + residual.double()
    return acc, (1.2 if act else 1.0) * 2.0 ** -15 * s


def _check(got, ref, extra, what, fp32=False):
    err = (got.double() - ref).abs()
    if fp32:
        tol = extra + 2.0 ** -22 * ref.abs()
    else:
        tol = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 10) + extra
    bad = ~(err <= tol)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {err.numel()} outside the bound, worst err {float(err.max()):.3e}"


@pytest.mark.parametrize("case", ["row_bias_silu", "col_bias_quick_gelu", "f32_residual"])
def test_epilogue_many_units_per_cta(native_lib, case):
    """M = 40,000 (ragged last row block) x N = 640: 313 x 5 output tiles of 128 x 128, about twelve per CTA"""
    from riffusion import tc_ops as ops

    M, N, K = 40000, 640, 640
    torch.manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV) * 0.5).half()
    b = (torch.randn(N, K, device=DEV) * K ** -0.5).half()
    kw, out_dtype = {
        "row_bias_silu": (dict(bias=torch.randn(M, device=DEV).half(), bias_per_row=True, act=ops.ACT_SILU), torch.float16),
        "col_bias_quick_gelu": (dict(bias=torch.randn(N, device=DEV).half(), act=ops.ACT_QUICK_GELU, alpha=1.5), torch.float16),
        "f32_residual": (dict(bias=torch.randn(N, device=DEV).half(), residual=torch.randn(M, N, device=DEV).half(),
                              alpha=0.5), torch.float32),
    }[case]
    got = ops.gemm(a, b, out_dtype=out_dtype, **kw).reshape(M, N)
    ref, acc_tol = _ref(a, b, **kw)
    _check(got, ref, acc_tol, case, fp32=out_dtype == torch.float32)


def test_split_k_partials_more_units_than_sms(native_lib, monkeypatch):
    """M = 1024, N = 1280, K = 11520: 8 x 10 tiles of 128 x 128 whose 180 K slabs are cut into splits (three on a
    132-SM H100), so some CTAs store the fp32 partials of more than one unit; column bias + residual applied by the
    second stage"""
    from riffusion import tc_ops as ops

    M, N, K = 1024, 1280, 11520
    requests = []
    orig = ops._workspace

    def spy(nbytes, desc, device):
        requests.append(int(nbytes))
        return orig(nbytes, desc, device)

    monkeypatch.setattr(ops, "_workspace", spy)
    torch.manual_seed(7)
    a = (torch.randn(M, K, device=DEV) * 0.5).half()
    b = (torch.randn(N, K, device=DEV) * K ** -0.5).half()
    bias = torch.randn(N, device=DEV).half()
    res = torch.randn(M, N, device=DEV).half()
    got = ops.gemm(a, b, bias=bias, residual=res).reshape(M, N)
    splits = requests[-1] // (M * N * 4)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert splits * 80 > sms, f"{splits} splits of 80 tiles do not exceed the {sms} SMs"
    ref, acc_tol = _ref(a, b, bias=bias, residual=res)
    _check(got, ref, acc_tol, "split-K")

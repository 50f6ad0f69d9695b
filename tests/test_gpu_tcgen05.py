"""wgmma GEMM with fused bias + GELU epilogue (csrc/gemm_wgmma.cu) against a plain PyTorch fp32 reference: ragged M,
both tile widths, K up to 3072, the full GPT-2 c_fc shape, the aux epilogues and autograd."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
# variants 0 (tile per CTA), 1 (persistent CTAs) and 2 (two-CTA clusters sharing W by TMA multicast); variant 3
# (persistent two-CTA clusters, column-sum output) is tested in tests/test_gpu_tcgen05_pp.py
VARIANTS = [int(v) for v in os.environ.get("ADAPCC_TCGEN05_TEST_VARIANTS", "0,1,2").split(",") if v.strip()]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


@pytest.mark.parametrize("m,n,k,act", [(128, 256, 64, "none"), (256, 256, 128, "gelu"), (200, 384, 192, "gelu"),
                                       (1024, 3072, 768, "gelu"), (384, 128, 3072, "none"),
                                       (8192, 3072, 768, "gelu")])
@pytest.mark.parametrize("variant", VARIANTS)
def test_gemm_bias_act_matches_fp32_reference(dev, m, n, k, act, variant):
    from adapcc_b200.ops.gemm import linear_act

    if variant == 2 and n % 256 != 0:
        pytest.skip("CTA-pair variant needs N % 256 == 0")
    torch.manual_seed(m + n + k)
    x = torch.randn(m, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
    b = torch.randn(n, device=dev).bfloat16()
    out, pre = linear_act(x, w, b, act, save_pre=True, variant=variant)
    torch.cuda.synchronize()
    u = x.float() @ w.float().t() + b.float()
    assert torch.allclose(pre.float(), u, atol=3e-2, rtol=2e-2), (pre.float() - u).abs().max()
    want = torch.nn.functional.gelu(u.bfloat16().float(), approximate="tanh") if act == "gelu" else u
    assert torch.allclose(out.float(), want, atol=3e-2, rtol=2e-2), (out.float() - want).abs().max()


def test_linear_gelu_autograd_matches_torch(dev):
    from adapcc_b200.ops.gemm import linear_gelu

    torch.manual_seed(3)
    x = torch.randn(4, 96, 256, device=dev).bfloat16().requires_grad_(True)
    w = (torch.randn(1024, 256, device=dev) / 16).bfloat16().requires_grad_(True)
    b = torch.randn(1024, device=dev).bfloat16().requires_grad_(True)
    dy = torch.randn(4, 96, 1024, device=dev).bfloat16()
    linear_gelu(x, w, b).backward(dy)
    xr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    torch.nn.functional.gelu(torch.nn.functional.linear(xr, wr, br), approximate="tanh").backward(dy.float())
    for got, want in ((x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
        err = (got.float() - want).abs().max() / want.abs().max()
        assert err < 3e-2, err


def test_aux_epilogues_and_fused_mlp(dev):
    from adapcc_b200.ops.gemm import linear_act, mlp_gelu

    torch.manual_seed(5)
    m, n, k = 384, 1024, 256
    x = torch.randn(m, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
    b = torch.randn(n, device=dev).bfloat16()
    aux = torch.randn(m, n, device=dev).bfloat16()
    acc = x.float() @ w.float().t()
    got, _ = linear_act(x, w, b, "residual", aux=aux)
    want = (acc + b.float()).bfloat16().float() + aux.float()
    assert torch.allclose(got.float(), want, atol=4e-2, rtol=2e-2)
    got, _ = linear_act(x, w, None, "dgelu", aux=aux)
    a = aux.float().requires_grad_(True)
    torch.nn.functional.gelu(a, approximate="tanh").sum().backward()
    assert torch.allclose(got.float(), acc * a.grad, atol=4e-2, rtol=3e-2)
    # whole MLP, both directions
    d, hid = 256, 1024
    xs = torch.randn(4, 96, d, device=dev).bfloat16().requires_grad_(True)
    w1 = (torch.randn(hid, d, device=dev) / 16).bfloat16().requires_grad_(True)
    b1 = torch.randn(hid, device=dev).bfloat16().requires_grad_(True)
    w2 = (torch.randn(d, hid, device=dev) / 32).bfloat16().requires_grad_(True)
    b2 = torch.randn(d, device=dev).bfloat16().requires_grad_(True)
    dy = torch.randn(4, 96, d, device=dev).bfloat16()
    mlp_gelu(xs, w1, b1, w2, b2).backward(dy)
    ref = [t.detach().float().requires_grad_(True) for t in (xs, w1, b1, w2, b2)]
    F = torch.nn.functional
    F.linear(F.gelu(F.linear(ref[0], ref[1], ref[2]), approximate="tanh"), ref[3], ref[4]).backward(dy.float())
    for got, want in zip((xs, w1, b1, w2, b2), ref):
        err = (got.grad.float() - want.grad).abs().max() / want.grad.abs().max()
        assert err < 3e-2, err

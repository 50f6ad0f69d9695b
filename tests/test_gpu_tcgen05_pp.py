"""wgmma GEMM variant 3 — persistent two-CTA clusters sharing the W slab by TMA multicast (csrc/gemm_wgmma.cu) —
against plain PyTorch fp32 references: identity / GELU(+pre) / dGELU(+column sums), ragged M, one to many tiles per
cluster, and the fused MLP autograd path built on it."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch.device("cuda:0")


@pytest.mark.parametrize("m,n,k,act", [(256, 256, 64, "none"), (256, 512, 128, "gelu"), (200, 256, 192, "gelu"),
                                       (1000, 768, 3072, "none"), (8192, 3072, 768, "gelu"), (40000, 256, 64, "gelu")])
def test_pp_gemm_matches_fp32_reference(dev, m, n, k, act):
    from adapcc_b200.ops.gemm import linear_act

    torch.manual_seed(m + n + k)
    x = torch.randn(m, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
    b = torch.randn(n, device=dev).bfloat16()
    out, pre = linear_act(x, w, b, act, save_pre=True, variant=3)
    torch.cuda.synchronize()
    u = x.float() @ w.float().t() + b.float()
    assert torch.allclose(pre.float(), u, atol=3e-2, rtol=2e-2), (pre.float() - u).abs().max()
    want = torch.nn.functional.gelu(u.bfloat16().float(), approximate="tanh") if act == "gelu" else u
    assert torch.allclose(out.float(), want, atol=3e-2, rtol=2e-2), (out.float() - want).abs().max()
    out2, none = linear_act(x, w, b, act, save_pre=False, variant=3)          # without the pre-activation output
    assert none is None and torch.equal(out2, out)


@pytest.mark.parametrize("m,n,k", [(384, 1024, 256), (8192, 3072, 768), (300, 256, 768)])
def test_pp_dgelu_and_colsum(dev, m, n, k):
    from adapcc_b200.ops.gemm import linear_act

    torch.manual_seed(7 + m)
    x = torch.randn(m, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
    aux = torch.randn(m, n, device=dev).bfloat16()
    acc = x.float() @ w.float().t()
    colsum = torch.zeros(n, dtype=torch.float32, device=dev)
    got, _ = linear_act(x, w, None, "dgelu", aux=aux, colsum=colsum, variant=3)
    a = aux.float().requires_grad_(True)
    torch.nn.functional.gelu(a, approximate="tanh").sum().backward()
    want = acc * a.grad
    assert torch.allclose(got.float(), want, atol=4e-2, rtol=3e-2), (got.float() - want).abs().max()
    ref_cs = got.float().sum(0)                                   # sums of the bf16 values the kernel wrote
    assert torch.allclose(colsum, ref_cs, atol=2e-2 * max(1.0, float(ref_cs.abs().max())), rtol=1e-2)
    for _ in range(3):                                            # the column sums are added in a fixed order
        again = torch.zeros_like(colsum)
        got2, _ = linear_act(x, w, None, "dgelu", aux=aux, colsum=again, variant=3)
        assert torch.equal(got2, got) and torch.equal(again, colsum)


def test_pp_fused_mlp_autograd(dev, monkeypatch):
    from adapcc_b200.ops.gemm import mlp_gelu

    monkeypatch.setenv("ADAPCC_TCGEN05_VARIANT", "3")
    torch.manual_seed(5)
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

"""Swish dual-output GEMM epilogue (feed-forward hidden layer): fp32 FFMA path vs float64, tf32 wgmma path vs fp32."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200.ops import call, gemm


def test_swish_dual_epilogue():
    M, K, N = 1500, 64, 256
    g = torch.Generator().manual_seed(3)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * 0.2, torch.randn(N, generator=g)
    seed, p = 99, 0.2
    thr, inv = ops.drop_params(p)
    mask = torch.empty(M * N, device=DEV)
    call("cmgan_dropout_mask", mask, M * N, seed, thr)
    keep = mask.view(M, N).double().cpu()
    h_ref = x.double() @ W.double().t() + b.double()
    a_ref = h_ref * torch.sigmoid(h_ref) * keep * inv
    outs = {}
    for prec in (0, 1):
        h = torch.zeros(M, N, device=DEV)
        a = torch.zeros(M, N, device=DEV)
        gemm(A=x.to(DEV), lda=K, W=W.to(DEV), sb_k=1, sb_n=K, bias=b.to(DEV), C=h, ldc=N, M=M, N=N, Cin=K, epi=ops.EPI_SWISH_DUAL, C2=a, ldc2=N,
             seed=seed, drop_p=p, precision=prec)
        a_only = torch.zeros(M, N, device=DEV)
        gemm(A=x.to(DEV), lda=K, W=W.to(DEV), sb_k=1, sb_n=K, bias=b.to(DEV), C=None, ldc=N, M=M, N=N, Cin=K, epi=ops.EPI_SWISH_DUAL, C2=a_only,
             ldc2=N, seed=seed, drop_p=p, precision=prec)
        torch.cuda.synchronize()
        assert torch.equal(a, a_only)
        outs[prec] = (h.double().cpu(), a.double().cpu())
    tol = {0: 3e-6, 1: 4e-3}
    for prec in (0, 1):
        for name, got, ref in (("h", outs[prec][0], h_ref), ("a", outs[prec][1], a_ref)):
            err = (got - ref).abs().max().item()
            print(f"[parity] swish-dual prec={prec} {name}: max-abs {err:.3e} (range {ref.abs().max().item():.3e})")
            assert err <= tol[prec] * ref.abs().max().item()


@pytest.mark.parametrize("B,T,Fw,axis", [(2, 321, 3, 0), (2, 5, 101, 1), (1, 530, 1, 0), (1, 4, 2, 0), (1, 70, 2, 0), (3, 2, 17, 1)])
def test_attention_fwd_tensor_core(B, T, Fw, axis):
    g = torch.Generator().manual_seed(7)
    M = B * T * Fw
    qkv = torch.randn(M, 192, generator=g).to(DEV)
    E = (torch.randn(1025, 16, generator=g) * 0.5).to(DEV)
    ref, lse_ref = torch.empty(M, 64, device=DEV), torch.empty(M, 4, device=DEV)
    got, lse = torch.full((M, 64), float("nan"), device=DEV), torch.full((M, 4), float("nan"), device=DEV)
    call("cmgan_attention_fwd", qkv, E, B, T, Fw, axis, ref, lse_ref)
    call("cmgan_attention_fwd_tf32", qkv, E, B, T, Fw, axis, got, lse)
    torch.cuda.synchronize()
    err = (got - ref).abs().max().item()
    lerr = (lse - lse_ref).abs().max().item()
    print(f"[parity-tf32] attention fwd axis={axis} L={T if axis == 0 else Fw}: ctx max-abs {err:.3e} (range {ref.abs().max().item():.2e}), lse {lerr:.3e}")
    assert np.isfinite(err) and err < 1e-2 * ref.abs().max().item() and lerr < 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize("B,T,Fw,axis", [(1, 70, 3, 0), (2, 5, 101, 1), (1, 321, 2, 0), (1, 3, 130, 1), (3, 64, 5, 0), (1, 700, 1, 0)])
def test_attention_bwd_tensor_core(B, T, Fw, axis):
    """tf32 mma.sync backward (dq / dk / dv / dE, skewed relative-position terms) vs the exact fp32 backward"""
    g = torch.Generator().manual_seed(11)
    M = B * T * Fw
    qkv = torch.randn(M, 192, generator=g).to(DEV)
    E = (torch.randn(1025, 16, generator=g) * 0.5).to(DEV)
    dctx = torch.randn(M, 64, generator=g).to(DEV)
    ctx, lse = torch.empty(M, 64, device=DEV), torch.empty(M, 4, device=DEV)
    call("cmgan_attention_fwd", qkv, E, B, T, Fw, axis, ctx, lse)
    out = {}
    for name in ("cmgan_attention_bwd", "cmgan_attention_bwd_tf32"):
        delta = torch.full((M, 4), float("nan"), device=DEV)
        dqkv = torch.full((M, 192), float("nan"), device=DEV)
        dE = torch.zeros(1025, 16, device=DEV)
        call(name, qkv, E, ctx, dctx, lse, B, T, Fw, axis, delta, dqkv, dE)
        torch.cuda.synchronize()
        out[name] = (dqkv, dE, delta)
    (r_dqkv, r_dE, r_dl), (g_dqkv, g_dE, g_dl) = out["cmgan_attention_bwd"], out["cmgan_attention_bwd_tf32"]
    L = T if axis == 0 else Fw
    for nm, got, ref in (("dq", g_dqkv[:, :64], r_dqkv[:, :64]), ("dk", g_dqkv[:, 64:128], r_dqkv[:, 64:128]),
                         ("dv", g_dqkv[:, 128:], r_dqkv[:, 128:]), ("dE", g_dE, r_dE), ("delta", g_dl, r_dl)):
        err = (got - ref).abs().max().item()
        scale = ref.abs().max().item()
        print(f"[parity-tf32] attention bwd axis={axis} L={L} {nm}: max-abs {err:.3e} (range {scale:.2e})")
        assert np.isfinite(err) and err < 1e-2 * scale, nm

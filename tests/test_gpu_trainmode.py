"""Parity of the path bench.py times: train mode (dropout with exported masks, BatchNorm batch statistics) in both precisions,
at the bench shapes, against the float64 oracle -- and the tf32 tensor-core backward kernels directly against float64 math.

Tolerances (relative to each tensor's max, floor 1e-3 of the largest gradient of the model where stated):
  fp32 mode: forward 2e-5, gradients 5e-3 (the reference's own fp32 backward is 2.8e-3 from float64 on the deepest layers);
  tf32 mode: tf32 keeps 10 mantissa bits (unit round-off 2^-11 = 4.9e-4 per operand): one contraction 1.5e-3, a conformer block
  forward 5e-3 / gradients 3e-2, the whole 60-layer network's parameter gradients 8e-2 (InstanceNorm / LayerNorm cancellations
  amplify the operand rounding; measured values are printed).
The float64 oracle runs on the GPU here (same code, torch CUDA float64 -- no TF32 involved) so that the bench shapes finish in seconds.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
if torch.cuda.is_available():
    import cmgan_b200
    from cmgan_b200 import conformer_block as G, network, ops, signal
    from cmgan_b200.ops import call, gemm
from oracle import cmgan_oracle as O
from tf32_model import tf32_rna, tf32_rz


def _rel(got, ref, floor=0.0):
    got, ref = got.detach().double(), ref.detach().double().to(got.device)
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs().max().item()
    return err / max(ref.abs().max().item(), floor, 1e-30)


def _rows_from_seq(x, B, T, F2, axis):
    Cn = x.shape[-1]
    if axis == 0:
        return x.view(B, F2, T, Cn).permute(0, 2, 1, 3).reshape(-1, Cn)
    return x.reshape(-1, Cn)


def _seq_from_rows(r, B, T, F2, axis):
    Cn = r.shape[-1]
    if axis == 0:
        return r.view(B, T, F2, Cn).permute(0, 2, 1, 3).reshape(B * F2, T, Cn)
    return r.view(B * T, F2, Cn)


def _block_masks(seed, block_id, prefix, B, T, F2, axis):
    """the five dropout masks conformer_fwd draws for this block (same counter-based generator), in the oracle's layout"""
    M = B * T * F2
    thr, _ = ops.drop_params(0.2)
    out = {}
    for site, (key, width) in enumerate([(".ff1.d1", 256), (".ff1.d2", 64), (".attn.d", 64), (".ff2.d1", 256), (".ff2.d2", 64)]):
        m = torch.empty(M * width, device=DEV)
        call("cmgan_dropout_mask", m, M * width, G._site_seed(seed, block_id, site), thr)
        out[prefix + key] = _seq_from_rows(m.view(M, width), B, T, F2, axis).double()
    return out


@pytest.fixture(scope="module")
def weights(g_weights):
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    return m.to(DEV)


# ------------------------------------------------------------------------------------------------ conformer block, train mode
@pytest.mark.parametrize("mode,axis,prefix,B,T,F2", [
    ("fp32", 0, "TSCB_1.time_conformer", 2, 37, 3), ("fp32", 1, "TSCB_3.freq_conformer", 2, 3, 37),
    ("tf32", 0, "TSCB_2.time_conformer", 2, 37, 3), ("tf32", 1, "TSCB_4.freq_conformer", 2, 3, 37),
    ("tf32", 0, "TSCB_1.time_conformer", 4, 321, 101), ("tf32", 1, "TSCB_1.freq_conformer", 4, 321, 101),     # the bench shape
    ("fp32", 0, "TSCB_4.time_conformer", 4, 321, 101)])
def test_conformer_block_train_mode(weights, g_weights, mode, axis, prefix, B, T, F2):
    """dropout (exported masks) + BatchNorm batch statistics + running-stat update, forward and backward, vs float64"""
    weights.load_state_dict(g_weights, strict=True)          # running statistics back to the checkpoint's
    P = weights._tensor_dict()
    g = torch.Generator().manual_seed(11)
    L = T if axis == 0 else F2
    N = B * F2 if axis == 0 else B * T
    xs = torch.randn(N, L, 64, generator=g)
    dy = torch.randn(N, L, 64, generator=g)
    seed, block_id = 77, 3
    masks = _block_masks(seed, block_id, prefix, B, T, F2, axis)
    sd64 = {k: (v.double().to(DEV).requires_grad_(True) if v.is_floating_point() else v.to(DEV)) for k, v in g_weights.items() if k.startswith(prefix)}
    xs64 = xs.double().to(DEV).requires_grad_(True)
    bn_out = {}
    ref = O.conformer_block(xs64, sd64, prefix, training=True, masks=masks, bn_out=bn_out) + xs64
    ref.backward(dy.double().to(DEV))
    ops.set_precision(mode)
    try:
        rows = _rows_from_seq(xs, B, T, F2, axis).contiguous().to(DEV)
        save = {}
        y = G.conformer_fwd(rows, P, prefix, B, T, F2, axis, True, seed, block_id, G._Sums(4096, DEV), save)
        grads = {k: torch.zeros_like(v) for k, v in P.items() if k.startswith(prefix) and v.is_floating_point()}
        dx = G.conformer_bwd(_rows_from_seq(dy, B, T, F2, axis).contiguous().to(DEV), save, P, grads, B, T, F2, G._Sums(4096, DEV))
        ops.join_wgrad()
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    # fp32 gradients: 5e-3 as for the whole network (the depthwise-conv bias in front of a train-mode BatchNorm has a mathematically zero
    # gradient: what is measured there is fp32 summation noise over 130 k rows against the 1e-3 x gmax floor)
    tol_f, tol_g = (2e-5, 5e-3) if mode == "fp32" else (5e-3, 3e-2)
    e_f = _rel(_seq_from_rows(y, B, T, F2, axis), ref)
    e_x = _rel(_seq_from_rows(dx, B, T, F2, axis), xs64.grad)
    # BatchNorm running statistics after one training forward (momentum 0.1, unbiased variance)
    mean_b, var_b = bn_out[prefix + ".conv"]
    rm0, rv0 = g_weights[prefix + ".conv.net.5.running_mean"].double().to(DEV), g_weights[prefix + ".conv.net.5.running_var"].double().to(DEV)
    e_rm = _rel(P[prefix + ".conv.net.5.running_mean"], 0.9 * rm0 + 0.1 * mean_b)
    e_rv = _rel(P[prefix + ".conv.net.5.running_var"], 0.9 * rv0 + 0.1 * var_b)
    gmax = max(v.grad.abs().max().item() for v in sd64.values() if v.is_floating_point() and v.grad is not None)
    worst, wk = 0.0, ""
    for k, v in sd64.items():
        if not v.is_floating_point() or v.grad is None or "running_" in k:
            continue
        e = _rel(grads[k], v.grad, floor=1e-3 * gmax)
        if e > worst:
            worst, wk = e, k
    print(f"[parity-train] {mode} {prefix} B={B} T={T} F'={F2}: fwd {e_f:.3e}  dx {e_x:.3e}  worst grad {worst:.3e} ({wk})  "
          f"running_mean {e_rm:.2e} running_var {e_rv:.2e}")
    assert e_f <= tol_f and e_x <= tol_g and worst <= tol_g, (e_f, e_x, worst, wk)
    assert e_rm <= 5e-3 and e_rv <= 5e-3


# ------------------------------------------------------------------------------------------------ whole network, train mode
def _net_masks(seed, B, T, F2):
    masks = {}
    for i in range(1, 5):
        for axis, name in ((0, "time_conformer"), (1, "freq_conformer")):
            masks.update(_block_masks(seed, (i - 1) * 2 + axis, f"TSCB_{i}.{name}", B, T, F2, axis))
    return masks


@pytest.mark.parametrize("mode,nsamp", [("fp32", 8000), ("tf32", 32000)])
def test_tscnet_train_mode_vs_oracle(g_weights, mode, nsamp):
    """TSCNet forward + backward in train mode (B = 2; 2 s clips in tf32 = the timed configuration's shapes) vs float64"""
    m = cmgan_b200.TSCNet(64, 201)
    m.load_state_dict(g_weights, strict=True)
    m = m.to(DEV).train()
    P = m._tensor_dict()
    gen = torch.Generator().manual_seed(3)
    clean = 0.05 * torch.randn(2, nsamp, generator=gen)
    noisy = (clean + 0.05 * torch.randn(2, nsamp, generator=gen)).to(DEV)
    x = signal.stft_compress(noisy, signal.rms_scale(noisy)).permute(0, 1, 3, 2)        # (B, 2, T, F)
    B, _, T, F = x.shape
    F2 = (F - 1) // 2 + 1
    seed = 5
    masks = _net_masks(seed, B, T, F2)
    sd = {k: (v.double().to(DEV).requires_grad_(True) if v.is_floating_point() and "running_" not in k else v.to(DEV)) for k, v in g_weights.items()}
    fr64, fi64 = O.tscnet_forward(x.double(), sd, training=True, masks=masks)
    (fr64.square().mean() + fi64.square().mean()).backward()
    ops.set_precision(mode)
    try:
        S = {}
        fr, fi = network.tscnet_fwd(x, P, True, seed, S)
        n = fr.numel()
        grads = {k: torch.zeros_like(v) for k, v in P.items() if v.is_floating_point() and "running_" not in k}
        network.tscnet_bwd(S, fr * (2.0 / n), fi * (2.0 / n), P, grads)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    e_r, e_i = _rel(fr, fr64), _rel(fi, fi64)
    gmax = max(sd[k].grad.abs().max().item() for k in grads if sd[k].grad is not None)
    worst, wk = 0.0, ""
    for k in grads:
        if sd[k].grad is None:
            continue
        e = _rel(grads[k], sd[k].grad, floor=1e-3 * gmax)
        if e > worst:
            worst, wk = e, k
    print(f"[parity-train] {mode} TSCNet train mode B=2 T={T}: final_real {e_r:.3e} final_imag {e_i:.3e}; worst parameter gradient {worst:.3e} ({wk})")
    rms = lambda a, b: ((a.double() - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()      # noqa: E731
    print(f"[parity-train] {mode} TSCNet train mode: relative rms error final_real {rms(fr, fr64):.3e} final_imag {rms(fi, fi64):.3e}")
    # tf32, train mode, 2 s: the max-abs deviation of the un-thresholded mask x magnitude output reaches ~1e-2 of the output range (rms 10x lower);
    # the same path in eval mode on real speech is 1.7e-4 abs / 73 dB SNR on the waveform (tests/test_gpu_audiosamples.py)
    tol_f, tol_g = (2e-4, 5e-3) if mode == "fp32" else (2.5e-2, 8e-2)
    assert e_r <= tol_f and e_i <= tol_f and worst <= tol_g, (e_r, e_i, worst, wk)
    assert rms(fr, fr64) <= tol_f / 4 and rms(fi, fi64) <= tol_f / 4


# ------------------------------------------------------------------------------------------------ tf32 kernels vs float64 directly
def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("M,K,N", [(129684, 64, 256), (129684, 256, 64), (5000, 128, 64), (129684, 192, 64)])
def test_tc_dgrad_gemm_vs_float64(M, K, N):
    """data-gradient form (weight read transposed) of the wgmma tf32 GEMM vs float64 on the same operands, and against its exact
    operand-rounding model: A is raw randn streamed by TMA, so the tensor core truncates it; the packed weight is rounded to nearest"""
    dy, W = _rand(M, K, seed=1), _rand(K, N, seed=2, scale=K ** -0.5)       # dx = dy @ W, W stored (K, N): sb_k = N, sb_n = 1
    out = torch.empty(M, N, device=DEV)
    gemm(A=dy, lda=K, W=W, sb_k=N, sb_n=1, C=out, ldc=N, M=M, N=N, Cin=K, precision=1)
    ref = dy.double() @ W.double()
    e = _rel(out, ref)
    e_rna = _rel(out, tf32_rna(dy).double() @ tf32_rna(W).double())
    e_rz = _rel(out, tf32_rz(dy).double() @ tf32_rna(W).double())
    print(f"[tf32-vs-f64] dgrad GEMM ({M}x{K})x({K}x{N}): vs float64 {e:.3e}; vs rna-rounded operands {e_rna:.3e}; vs truncated A {e_rz:.3e}")
    assert e <= 1.5e-3
    assert e_rz <= 2e-5, "the kernel must equal a float64 product of truncated A and rounded W up to fp32 accumulation"


@pytest.mark.parametrize("M,K,N,dil", [(129684, 64, 256, 0), (129684, 256, 64, 0), (4 * 321 * 101, 128, 64, 2)])
def test_tc_wgrad_vs_float64(M, K, N, dil):
    """weight-gradient kernels in tf32 mode (dense and dilated-convolution gather) vs float64"""
    if dil == 0:
        x, dy = _rand(M, K, seed=3), _rand(M, N, seed=4)
        dW, db = torch.zeros(N, K, device=DEV), torch.zeros(N, device=DEV)
        gemm(wgrad=True, A=x, lda=K, Cin=K, D=dy, ldd=N, N=N, W=None, C=dW, sb_k=1, sb_n=K, ldc=0, M=M, dbias=db, precision=1)
        ops.join_wgrad()
        ref = dy.double().t() @ x.double()
        e_b = _rel(db, dy.double().sum(0))
    else:
        B, T, Fw = 4, 321, 101
        cat, dy = _rand(M, 320, seed=5), _rand(M, N, seed=6)
        c0 = 320 - K
        taps = network._dense_taps(dil)
        dW, db = torch.zeros(N, K, 2, 3, device=DEV), torch.zeros(N, device=DEV)
        gemm(wgrad=True, A=(cat, c0), lda=320, Cin=K, taps=taps, conv=dict(OH=T, OW=Fw, IH=T, IW=Fw), D=dy, ldd=N, N=N, W=None, C=dW, sb_tap=1, sb_k=6,
             sb_n=K * 6, ldc=0, M=M, dbias=db, precision=1)
        ops.join_wgrad()
        xin = cat[:, c0:].double().view(B, T, Fw, K).permute(0, 3, 1, 2)
        g = dy.double().view(B, T, Fw, N).permute(0, 3, 1, 2)
        xp = torch.nn.functional.pad(xin, (1, 1, dil, 0))
        ref = torch.nn.grad.conv2d_weight(xp, (N, K, 2, 3), g, dilation=(dil, 1))
        e_b = _rel(db, dy.double().sum(0))
    e = _rel(dW, ref)
    print(f"[tf32-vs-f64] wgrad M={M} K={K} N={N} dil={dil}: dW {e:.3e}, dbias {e_b:.3e}")
    assert e <= 2e-3 and e_b <= 2e-3


def _attn_ref64(qkv, E, B, T, F2, axis):
    """float64 attention core on channel-last rows: returns ctx rows (autograd-enabled)"""
    Cn = 64
    q, k, v = (_seq_from_rows(qkv[:, i * Cn:(i + 1) * Cn], B, T, F2, axis) for i in range(3))
    N, L, _ = q.shape
    q, k, v = (t.view(N, L, 4, 16).permute(0, 2, 1, 3) for t in (q, k, v))
    seq = torch.arange(L, device=qkv.device)
    dist = (seq.view(L, 1) - seq.view(1, L)).clamp(-512, 512) + 512
    dots = (q @ k.transpose(-1, -2)) * 0.25 + torch.einsum("bhnd,nrd->bhnr", q, E[dist]) * 0.25
    out = (torch.softmax(dots, -1) @ v).permute(0, 2, 1, 3).reshape(N, L, Cn)
    return _rows_from_seq(out, B, T, F2, axis)


@pytest.mark.parametrize("fwd", ["cmgan_attention_fwd_tf32"])
@pytest.mark.parametrize("B,T,F2,axis", [(2, 321, 5, 0), (2, 7, 101, 1), (1, 641, 3, 0), (1, 1281, 2, 0), (3, 130, 2, 0), (1, 2, 64, 1),
                                         (2, 101, 4, 0), (1, 3, 321, 1), (2, 200, 3, 0), (1, 4, 129, 1), (1, 513, 2, 0), (2, 33, 7, 1)])
def test_tc_attention_fwd_bwd_vs_float64(B, T, F2, axis, fwd):
    """tensor-core attention forward and backward (dq, dk, dv, dE) directly vs float64 autograd, L = 321 / 101 / 641 / 1281"""
    M = B * T * F2
    qkv, E = _rand(M, 192, seed=7), _rand(1025, 16, seed=8, scale=0.5)
    dctx = _rand(M, 64, seed=9)
    q64, E64 = qkv.double().requires_grad_(True), E.double().requires_grad_(True)
    ref = _attn_ref64(q64, E64, B, T, F2, axis)
    ref.backward(dctx.double())
    ctx, lse = torch.empty(M, 64, device=DEV), torch.empty(M, 4, device=DEV)
    call(fwd, qkv, E, B, T, F2, axis, ctx, lse)
    dqkv, delta, dE = torch.empty(M, 192, device=DEV), torch.empty(M, 4, device=DEV), torch.zeros(1025, 16, device=DEV)
    call("cmgan_attention_bwd_tf32", qkv, E, ctx, dctx, lse, B, T, F2, axis, delta, dqkv, dE)
    e_c, e_q, e_e = _rel(ctx, ref), _rel(dqkv, q64.grad), _rel(dE, E64.grad)
    print(f"[tf32-vs-f64] attention ({fwd[16:]} forward) B={B} T={T} F'={F2} axis={axis}: ctx {e_c:.3e}  dqkv {e_q:.3e}  dE {e_e:.3e}")
    assert e_c <= 3e-3 and e_q <= 5e-3 and e_e <= 5e-3
    # same backward with the dE accumulators in a global scratch (3 blocks / SM variant of the dq kernel)
    from cmgan_b200._lib import lib
    nws = lib().cdll.cmgan_attention_bwd_ws_floats(B, T, F2, axis)
    ws = torch.empty(nws, device=DEV)
    dqkv2, dE2 = torch.empty(M, 192, device=DEV), torch.zeros(1025, 16, device=DEV)
    call("cmgan_attention_bwd_tf32_ws", qkv, E, ctx, dctx, lse, B, T, F2, axis, delta, dqkv2, dE2, 7, ws, nws)
    e_q2, e_e2 = _rel(dqkv2, q64.grad), _rel(dE2, E64.grad)
    print(f"[tf32-vs-f64] attention backward, global dE scratch: dqkv {e_q2:.3e}  dE {e_e2:.3e}")
    assert e_q2 <= 5e-3 and e_e2 <= 5e-3


# ------------------------------------------------------------------------------------------------ fused feed-forward kernel
@pytest.mark.parametrize("M,p_drop", [(129684, 0.2), (129684, 0.0), (300, 0.2), (128 * 148 * 2 + 77, 0.2)])
def test_fused_ffn_forward_vs_float64(g_weights, M, p_drop):
    """cmgan_ffn_fwd (LN -> W1 -> swish, dropout -> W2 -> dropout, 0.5, residual in one wgmma kernel) vs float64 with the exported masks"""
    pre = "TSCB_2.freq_conformer.ff1"
    w = {k[len(pre) + 1:]: v.to(DEV) for k, v in g_weights.items() if k.startswith(pre + ".")}
    x = _rand(M, 64, seed=21)
    s1, s2 = 1234567, 7654321
    thr, inv = ops.drop_params(p_drop)
    m1, m2 = torch.ones(M * 256, device=DEV), torch.ones(M * 64, device=DEV)
    if p_drop > 0:
        call("cmgan_dropout_mask", m1, M * 256, s1, thr)
        call("cmgan_dropout_mask", m2, M * 64, s2, thr)
    out = torch.empty(M, 64, device=DEV)
    W1, W2 = w["fn.fn.net.0.weight"], w["fn.fn.net.3.weight"]
    call("cmgan_ffn_fwd", x, 64, M, w["fn.norm.weight"], w["fn.norm.bias"], ops.packed_weight(W1, 0, 1, 64, 64, 1, 256), w["fn.fn.net.0.bias"],
         ops.packed_weight(W2, 0, 1, 256, 256, 1, 64), w["fn.fn.net.3.bias"], 0.5, s1, s2, thr, inv, None, out, 64)
    torch.cuda.synchronize()
    x64 = x.double()
    xn = torch.nn.functional.layer_norm(x64, (64,), w["fn.norm.weight"].double(), w["fn.norm.bias"].double(), 1e-5)
    h = xn @ W1.double().t() + w["fn.fn.net.0.bias"].double()
    a = h * torch.sigmoid(h) * m1.view(M, 256).double() * inv
    ref = x64 + 0.5 * (a @ W2.double().t() + w["fn.fn.net.3.bias"].double()) * m2.view(M, 64).double() * inv
    e = _rel(out - x, ref - x64)            # error of the branch itself (the residual would hide it)
    e_tot = _rel(out, ref)
    print(f"[fused-ffn] M={M} p={p_drop}: branch rel err {e:.3e}, output rel err {e_tot:.3e}")
    assert e <= 3e-3 and e_tot <= 1e-3


@pytest.mark.parametrize("M,p_drop,with_res2", [(129684, 0.2, True), (129684, 0.0, False), (300, 0.2, False), (128 * 148 + 5, 0.2, True)])
def test_fused_ffn_backward_vs_float64(g_weights, M, p_drop, with_res2):
    """cmgan_ffn_bwd (recompute of the hidden activation, dh in the same kernel, then dLN and the LayerNorm backward) vs float64 autograd of the
    same module with the exported mask; also the operands it leaves for the weight-gradient GEMMs (a, dh, xn)"""
    pre = "TSCB_3.time_conformer.ff2"
    w = {k[len(pre) + 1:]: v.to(DEV) for k, v in g_weights.items() if k.startswith(pre + ".")}
    x, dout = _rand(M, 64, seed=31), _rand(M, 64, seed=32)
    res2 = _rand(M, 64, seed=33) if with_res2 else None
    s1, s2 = 424242, 535353
    thr, inv = ops.drop_params(p_drop)
    m1, m2 = torch.ones(M * 256, device=DEV), torch.ones(M * 64, device=DEV)
    if p_drop > 0:
        call("cmgan_dropout_mask", m1, M * 256, s1, thr)
        call("cmgan_dropout_mask", m2, M * 64, s2, thr)
    m1, m2 = m1.view(M, 256).double() * inv, m2.view(M, 64).double() * inv
    W1, W2 = w["fn.fn.net.0.weight"], w["fn.fn.net.3.weight"]
    # float64 reference with autograd
    x64 = x.double().requires_grad_(True)
    g64, b64 = w["fn.norm.weight"].double().requires_grad_(True), w["fn.norm.bias"].double().requires_grad_(True)
    xn64 = torch.nn.functional.layer_norm(x64, (64,), g64, b64, 1e-5)
    xn64.retain_grad()
    h64 = xn64 @ W1.double().t() + w["fn.fn.net.0.bias"].double()
    h64.retain_grad()
    a64 = h64 * torch.sigmoid(h64) * m1
    out64 = x64 + 0.5 * (a64 @ W2.double().t() + w["fn.fn.net.3.bias"].double()) * m2
    out64.backward(dout.double())
    # the kernel's inputs: dz = 0.5 * mask2 * dout (rounded to tf32 by its producer)
    dz = tf32_rna((0.5 * m2 * dout.double()).float())
    dx = torch.empty(M, 64, device=DEV)
    a, dh, xn = torch.empty(M, 256, device=DEV), torch.empty(M, 256, device=DEV), torch.empty(M, 64, device=DEV)
    dg, db = torch.zeros(64, device=DEV), torch.zeros(64, device=DEV)
    call("cmgan_ffn_bwd", x, 64, dz, 64, dout, 64, res2, 64 if with_res2 else 0, M, w["fn.norm.weight"], w["fn.norm.bias"],
         ops.packed_weight(W1, 0, 1, 64, 64, 1, 256), w["fn.fn.net.0.bias"], ops.packed_weight(W2, 0, 256, 1, 64, 1, 256),
         ops.packed_weight(W1, 0, 64, 1, 256, 1, 64), s1, thr, inv, None, dx, 64, a, dh, xn, dg, db, torch.empty(M * 66, device=DEV))
    torch.cuda.synchronize()
    ref_dx = x64.grad + (res2.double() if with_res2 else 0.0)
    e_dx = _rel(dx - dout - (res2 if with_res2 else 0.0), ref_dx - dout.double() - (res2.double() if with_res2 else 0.0))     # the LayerNorm-backward branch itself
    e_a, e_dh, e_xn = _rel(a, a64), _rel(dh, h64.grad), _rel(xn, xn64)
    e_g, e_b = _rel(dg, g64.grad), _rel(db, b64.grad)
    print(f"[fused-ffn-bwd] M={M} p={p_drop}: dx branch {e_dx:.3e}  a {e_a:.3e}  dh {e_dh:.3e}  xn {e_xn:.3e}  dgamma {e_g:.3e}  dbeta {e_b:.3e}")
    assert e_dx <= 4e-3 and e_a <= 2e-3 and e_dh <= 3e-3 and e_xn <= 1e-3 and e_g <= 3e-3 and e_b <= 3e-3

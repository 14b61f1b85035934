"""Float64 checks of the tf32 tensor-core attention (csrc/attention_mma.cu) and the fused feed-forward (csrc/ffn_fused.cu), one C entry
point at a time.

The conventions are those of test_gpu_dense_f64.py (helpers in f64_check.py): guarded output buffers, NaN-filled overwrite-only outputs,
randomly prefilled accumulators (dE, dgamma, dbeta), and element-wise bounds |got - ref| <= c 2^-24 ref_abs.  Every bound here has terms
of very different size, so ref_abs is the whole bound in units of 2^-24 and c = 1; the comment next to each bound lists its terms.
References are float64 torch on the GPU, with autograd for the gradients, on the raw float32 inputs: the tf32 operand rounding is a term
of the bound, not part of the reference.

Where the kernels round (read from the code; a term per rounding point, in units of 2^-24 relative to the operand):
  TR = 2^13  rounded to nearest tf32 (cvt.rna, or tf32q's add-half-and-truncate): half a tf32 spacing
  TT = 2^14  truncated by the tensor core (raw fp32 staged by cp.async): a whole tf32 spacing
  - attention forward and dq kernel: q 0.25 log2(e) and dO rounded; K, V and the E window truncated; P and dS tf32q; ctx, dq stored rounded.
  - dk / dv kernel: K 0.25 log2(e) and V rounded; Q, dO and the E window truncated, and R2 = (Q 0.25 log2 e) E^T takes its Q operand
    unrounded, so it is truncated too: its logits differ from the forward's at the tf32 level.  P and dS tf32q; dk, dv stored rounded.
  - fused feed-forward: xn, the hidden a, dh and the packed W1 / W2 images rounded; dz is a tf32 operand by contract.
The float32 accumulation of a tensor-core sum grows by about 2^-24 per k-step (DESIGN.md section 4): a chain of K terms is charged K.
Where a softmax's sensitivity to its logits enters (ctx, lse, every gradient), the logits' error feeds p through eps_f / eps_b as in
test_attention_fp32, now with the tf32 operand terms.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from f64_check import DEV, EPS, NAN, SENT, U, _buf, _cdiv, _close, _close_tf32, _exact, _f32, _keep, _mix_seed, _randn, _swish_terms, _tail
from tf32_model import tf32_rna

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from cmgan_b200 import ops
    from cmgan_b200._lib import lib
    from cmgan_b200.ops import call

TR = 2.0 ** 13
TT = 2.0 ** 14
LOG2E = 1 / math.log(2)


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ================================================================================================ attention
def _seqs(t, B, T, Fw, axis):
    """(M, C) rows -> (S, L, C)"""
    C = t.shape[-1]
    t = t.reshape(B, T, Fw, C)
    return t.permute(0, 2, 1, 3).reshape(B * Fw, T, C) if axis == 0 else t.reshape(B * T, Fw, C)


def _rows(t, B, T, Fw, axis):
    """(S, L, C) -> (M, C)"""
    C = t.shape[-1]
    return (t.reshape(B, Fw, T, C).permute(0, 2, 1, 3) if axis == 0 else t.reshape(B, T, Fw, C)).reshape(-1, C)


def _heads(t):
    S, L, _ = t.shape
    return t.reshape(S, L, 4, 16).permute(0, 2, 1, 3)          # (S, 4, L, 16)


def _scores(q, k, E, dist):
    """0.25 q (k_j + E[clamp(i - j) + 512]) for (S, 4, L, 16) q, k"""
    return 0.25 * (q @ k.transpose(-1, -2) + torch.einsum("shid,ijd->shij", q, E[dist]))


def _dq_plan(L, n_items, per_sm):
    """mirror of dq_blocks in attention_mma.cu: (grid x, items per block) of the dq / dE kernel"""
    ntile = _cdiv(L, 64)
    gx = min(max(1, _nsm() * per_sm // ntile), n_items)
    return gx, _cdiv(n_items, gx)


def _attn_ref(qkv, E, dO, B, T, Fw, axis, dE_chain=None):
    """float64 attention on the GPU and the element-wise bounds of the tf32 kernels (units of 2^-24), as rows.  With dO also delta, dqkv and
    dE (their bounds need the dq kernel's plan: dE_chain = (sequential adds into one dE element, atomics into one dE element))."""
    sq = _seqs(qkv.double().to(DEV), B, T, Fw, axis)
    S, L = sq.shape[0], sq.shape[1]
    ql, kl, vl = (_heads(sq[..., 64 * i:64 * i + 64]).clone().requires_grad_() for i in range(3))
    El = E.double().to(DEV).requires_grad_()
    ar = torch.arange(L, device=DEV)
    dist = (ar[:, None] - ar[None, :]).clamp(-512, 512) + 512
    s = _scores(ql, kl, El, dist)
    p = torch.softmax(s, -1)
    cref = p @ vl
    R = {}
    rows = lambda t: _rows(t.permute(0, 2, 1, 3).reshape(S, L, -1), B, T, Fw, axis)          # (S, 4, L, c) -> (M, 4 c)
    rows4 = lambda t: _rows(t.permute(0, 2, 1).reshape(S, L, 4), B, T, Fw, axis)             # (S, 4, L) -> (M, 4)
    with torch.no_grad():
        qa, ka, va, Ea = (t.detach().abs() for t in (ql, kl, vl, El))
        a = _scores(qa, ka, Ea, dist)                                        # the score on absolute values (natural units)
        a_qk = 0.25 * qa @ ka.transpose(-1, -2)
        amax = a.max(-1, keepdim=True).values
        # forward / dq-kernel logits: q 0.25 log2 e rounded (TR + 1), K and E truncated (TT), 16-product mma sums (20); s - m and ex2 (2 amax + 4)
        e_f = (TR + 1 + TT + 20) * a + 2 * amax + 4
        eps_f = torch.expm1(U * e_f) / U                                     # relative error of one exponential, to all orders
        pe = p.detach() * eps_f
        spe = pe.sum(-1, keepdim=True)
        ca = cref.detach().abs()
        c1 = L + L / 8 + 4                                                   # sequential sums over the key tiles, the online rescale, 1 / l
        # ctx = sum tf32q(p) V_trunc / sum p: the chain and P's (TR) and V's (TT) rounding on every term; the exponentials' errors enter
        # numerator and denominator, sum p eps (|v| + |ctx|), over the perturbed denominator
        pv = p.detach() @ va
        lim_ctx = (c1 + TR + TT) * pv + (pe @ va + ca * spe) / (1 - U * spe).clamp_min(0.5)
        R["ctx"], R["lim_ctx"] = rows(cref.detach()), rows(lim_ctx)
        del e_f, eps_f, pe                                                   # full (S, 4, L, L) tensors: keep the peak low
        lse_n = torch.logsumexp(s.detach(), -1)
        # lse = m + log2 l (log2 units): the sum's chain and the logits' errors (log(1 + sum p eps) <= sum p eps), log2f and the add
        lim_lse = LOG2E * (c1 + spe.squeeze(-1)) + 2 * (amax.squeeze(-1) * LOG2E + math.log2(L) + 1) + (lse_n * LOG2E).abs()
        R["lse"], R["lim_lse"] = rows4(lse_n * LOG2E), rows4(lim_lse)
    if dO is None:
        return R
    do = _heads(_seqs(dO.double().to(DEV), B, T, Fw, axis))
    cref.backward(do)
    with torch.no_grad():
        da = do.abs()
        dref = (do * cref.detach()).sum(-1)
        # delta = sum dO ctx over the kernel's ctx (raw dO, 16 fmas): ctx's bound and its tf32 rounding, the chain
        lim_delta = (da * (lim_ctx + TR * ca)).sum(-1) + 17 * (da * ca).sum(-1)
        R["delta"], R["lim_delta"] = rows4(dref), rows4(lim_delta)
        # backward logits: the dk / dv kernel's are the larger -- K 0.25 log2 e rounded (TR + 1) and Q truncated (TT) on q.k, Q 0.25 log2 e
        # and E both truncated (2 TT + 1) on q.E -- then p = exp2(s - lse) with the forward's lse: its bound (ln 2 lim_lse), s - lse and ex2
        e_b = (TR + 1 + TT + 20) * a_qk + (2 * TT + 1 + 20) * (a - a_qk) + 2 * amax + 4 + \
            math.log(2) * lim_lse.unsqueeze(-1) + lse_n.abs().unsqueeze(-1) + 2
        eps_b = torch.expm1(U * e_b) / U
        dp = do @ vl.detach().transpose(-1, -2)
        dp_abs = da @ va.transpose(-1, -2)
        ddp = (dp - dref.unsqueeze(-1)).abs()
        pd = p.detach()
        ds = pd * (dp - dref.unsqueeze(-1))
        # ds = tf32q(p (dp - delta)): p's error, tf32q (TR) and two float32 roundings on |p (dp - delta)|; dp = dO V^T with one operand
        # rounded and one truncated (TR + TT) and 16 products; delta's bound
        dds = pd * ddp * (eps_b + TR + 2) + pd * ((TR + TT + 16) * dp_abs + lim_delta.unsqueeze(-1))
        # dv = sum_i tf32q(p_ij) dO_trunc,i: p's error, tf32q (TR), dO truncated (TT), the chain of L products
        lim_v = (pd * (eps_b + TR + TT + L + 2)).transpose(-1, -2) @ da
        del a, a_qk, e_b, eps_b, dp, dp_abs, ddp
    # dq = 0.25 (dS K_trunc + dR E_trunc), dk = 0.25 dS^T Q_trunc: linear in ds -- the gradients of the score on absolute values at ds's error
    # plus the truncated operand (TT) and the chain (2 L products for dq)
    qg, kg = (t.detach().abs().requires_grad_() for t in (ql, kl))
    _scores(qg, kg, Ea, dist).backward(dds + (TT + 2 * L + 8) * ds.abs())
    R["dqkv"] = torch.cat([rows(t.grad) for t in (ql, kl, vl)], -1)
    R["lim_dqkv"] = torch.cat([rows(qg.grad), rows(kg.grad), rows(lim_v)], -1)
    # dE = LN2 sum dR^T Qs, Qs = q 0.25 log2 e rounded (TR + 1): ds's error, the chain of sequential adds (per 64-query tile, per key tile
    # and item of a block, per atomic) and LN2 (2); the prefill is rounded once per atomic into its element
    n_seq, n_atom = dE_chain
    Eb = El.detach().abs().requires_grad_()
    _scores(qg.detach(), kg.detach(), Eb, dist).backward(dds + (TR + 1 + n_seq + n_atom + 2) * ds.abs())
    R["dE"], R["lim_dE"], R["n_atom"] = El.grad.reshape(-1), Eb.grad.reshape(-1), n_atom
    return R


def _attn_inputs(M, qscale, seed):
    qkv = _randn(M, 192, seed=seed)
    qkv[:, :64] *= qscale
    return qkv, _randn(1025, 16, seed=seed + 1, scale=0.5), _randn(M, 64, seed=seed + 2)


def _run_bwd(qd, Ed, ctx, dOd, lse, B, T, Fw, axis, M, how, dE0):
    """one backward as production issues it: 'parts7' (shared-memory dE), 'parts7_ws' (global dE scratch), 'split' (1, 4, 2 with the
    scratch: conformer_block's order).  -> (delta, dqkv, dE) guarded buffers"""
    delta, dqkv, dE = _buf(M * 4), _buf(M * 192), _buf(1025 * 16, dE0)
    nws = lib().cdll.cmgan_attention_bwd_ws_floats(B, T, Fw, axis)
    ws = _buf(nws)                                   # NaN: the dq kernel must zero its slabs
    args = (qd, Ed, ctx, dOd, lse, B, T, Fw, axis, delta, dqkv, dE)
    if how == "parts7":
        call("cmgan_attention_bwd_tf32_ws", *args, 7, None, 0)
    elif how == "parts7_ws":
        call("cmgan_attention_bwd_tf32_ws", *args, 7, ws, nws)
    else:
        call("cmgan_attention_bwd_tf32_ws", *args, 1, None, 0)
        call("cmgan_attention_bwd_tf32_ws", *args, 4, None, 0)
        call("cmgan_attention_bwd_tf32_ws", *args, 2, ws, nws)
    _tail(ws, nws, f"attention scratch ({how})")
    return delta, dqkv, dE


ATTN_L = [1, 2, 8, 15, 63, 64, 65, 127, 128, 129, 512, 513, 514, 600, 1281]
# (L, axis, q scale, B, other): two sequences' worth per axis at every L, peaked logits (q x 8); and plans where the dq kernel's blocks
# walk several (sequence, head) items in both variants (S = 64 at L = 65, S = 24 at L = 321)
ATTN_CASES = [(L, axis, qs, 2, 2) for L in ATTN_L for axis in (0, 1) for qs in (1.0, 8.0)] + \
             [(65, 0, 1.0, 2, 32), (65, 1, 8.0, 2, 32), (321, 0, 8.0, 2, 12), (321, 1, 1.0, 2, 12)]


@pytest.mark.parametrize("L,axis,qscale,B,other", ATTN_CASES)
def test_attention_tf32(L, axis, qscale, B, other):
    T, Fw = (L, other) if axis == 0 else (other, L)
    M, S = B * T * Fw, B * other
    n_items = 4 * S
    multi = other > 2
    (gx2, ipb2), (gx3, ipb3) = _dq_plan(L, n_items, 2), _dq_plan(L, n_items, 3)
    if multi:
        assert ipb2 > 1 and ipb3 > 1, f"the plan gives one item per block ({ipb2}, {ipb3}): the cross-item path is not reached"
    qkv, E, dO = _attn_inputs(M, qscale, 700)
    qd, Ed, dOd = qkv.to(DEV), E.to(DEV), dO.to(DEV)
    nm = f"L={L} axis={axis} q x{qscale:g} S={S}"

    # ---- forward: the default entry (single-buffered), the double-buffered instance, and lse = NULL
    ctx, lse = _buf(M * 64), _buf(M * 4)
    call("cmgan_attention_fwd_tf32", qd, Ed, B, T, Fw, axis, ctx, lse)
    ctx2, lse2 = _buf(M * 64), _buf(M * 4)
    call("cmgan_attention_fwd_tf32_nbuf", qd, Ed, B, T, Fw, axis, ctx2, lse2, 2)
    ctx3 = _buf(M * 64)
    call("cmgan_attention_fwd_tf32", qd, Ed, B, T, Fw, axis, ctx3, None)
    for b, n, what in ((ctx, M * 64, "ctx"), (lse, M * 4, "lse"), (ctx2, M * 64, "ctx nbuf 2"), (lse2, M * 4, "lse nbuf 2"), (ctx3, M * 64, "ctx lse=NULL")):
        _tail(b, n, f"attention fwd {what}")
    _exact(ctx2[:M * 64], ctx[:M * 64].cpu(), f"attention ctx nbuf 2 vs 1 {nm}")
    _exact(lse2[:M * 4], lse[:M * 4].cpu(), f"attention lse nbuf 2 vs 1 {nm}")
    _exact(ctx3[:M * 64], ctx[:M * 64].cpu(), f"attention ctx with lse = NULL {nm}")

    # dE's chain: per block 64-query mma sums into the accumulator, one add per key tile and item, one atomic per block row (clamped
    # distances: one per distance beyond 512 too)
    ntile = _cdiv(L, 64)
    n_atom = max(gx2, gx3) * ntile * max(1, L - 511)
    R = _attn_ref(qkv, E, dO, B, T, Fw, axis, dE_chain=(64 + max(ipb2, ipb3) * ntile + 4, n_atom))
    _close_tf32(ctx[:M * 64], R["ctx"].reshape(-1), R["lim_ctx"].reshape(-1), f"attention ctx {nm}")
    _close(lse[:M * 4], R["lse"].reshape(-1), R["lim_lse"].reshape(-1), 1, f"attention lse {nm}")

    # ---- delta alone (part 1): nothing else is touched
    dE0 = _randn(1025 * 16, seed=703)
    delta, dqkv, dE = _buf(M * 4), _buf(M * 192), _buf(1025 * 16, dE0)
    call("cmgan_attention_bwd_tf32_parts", qd, Ed, ctx, dOd, lse, B, T, Fw, axis, delta, dqkv, dE, 1)
    _close(delta[:M * 4], R["delta"].reshape(-1), R["lim_delta"].reshape(-1), 1, f"attention delta {nm}")
    _tail(delta, M * 4, "attention delta")
    assert bool(torch.isnan(dqkv[:M * 192]).all()), "part 1 wrote dqkv"
    _exact(dE[:1025 * 16], dE0, "part 1 changed dE")

    # ---- the three backward calls: dqkv bit-identical (no atomics touch it), dE bounded in each
    ref_dE = dE0.double() + R["dE"].cpu()
    lim_dE = dE0.double().abs() * (R["n_atom"] + 1) + R["lim_dE"].cpu()
    first = None
    for how in ("parts7", "parts7_ws", "split"):
        d, q, e = _run_bwd(qd, Ed, ctx, dOd, lse, B, T, Fw, axis, M, how, dE0)
        _tail(q, M * 192, f"attention dqkv ({how})")
        _tail(e, 1025 * 16, f"attention dE ({how})")
        _exact(d[:M * 4], delta[:M * 4].cpu(), f"attention delta ({how})")
        if first is None:
            first = q[:M * 192].cpu()
            _close_tf32(q[:M * 192], R["dqkv"].reshape(-1), R["lim_dqkv"].reshape(-1), f"attention dqkv {nm}")
        else:
            _exact(q[:M * 192], first, f"attention dqkv {how} vs parts7 {nm}")
        _close(e[:1025 * 16], ref_dE, lim_dE, 1, f"attention dE ({how}) {nm}")


@pytest.mark.parametrize("axis", [0, 1])
def test_attention_tf32_ragged(axis):
    """valid rows of every utterance within that utterance's own bound; rows t >= T_b of ctx and lse are left unwritten (NaN)"""
    frames = [1, 64, 65, 130, 600] if axis == 0 else [1, 4, 2, 5]
    B, T = len(frames), max(frames)
    Fw = 3 if axis == 0 else 129
    M = B * T * Fw
    qkv, E, _ = _attn_inputs(M, 4.0, 710)
    valid = torch.zeros(B, T, Fw, dtype=torch.bool)
    for b, tb in enumerate(frames):
        valid[b, :tb] = True
    valid = valid.reshape(-1)
    qkv[~valid] = NAN                                 # padding frames are never read
    ctx, lse = _buf(M * 64), _buf(M * 4)
    call("cmgan_attention_fwd_tf32_ragged", qkv.to(DEV), E.to(DEV), B, T, Fw, axis, torch.tensor(frames, dtype=torch.int32, device=DEV), ctx,
         lse)
    _tail(ctx, M * 64, "ragged ctx")
    _tail(lse, M * 4, "ragged lse")
    c, l = ctx[:M * 64].view(B, T, Fw, 64).cpu(), lse[:M * 4].view(B, T, Fw, 4).cpu()
    for b, tb in enumerate(frames):
        R = _attn_ref(qkv.view(B, T, Fw, 192)[b, :tb].reshape(-1, 192), E, None, 1, tb, Fw, axis)
        nm = f"ragged axis={axis} T_b={tb}"
        _close_tf32(c[b, :tb].reshape(-1), R["ctx"].reshape(-1), R["lim_ctx"].reshape(-1), f"attention ctx {nm}")
        _close(l[b, :tb].reshape(-1), R["lse"].reshape(-1), R["lim_lse"].reshape(-1), 1, f"attention lse {nm}")
        assert bool(torch.isnan(c[b, tb:]).all()) and bool(torch.isnan(l[b, tb:]).all()), f"{nm}: a row t >= T_b was written"


# ================================================================================================ fused feed-forward
def _ffn_x(M, seed):
    """rows of 64 channels: random rows, rows at mean / std = 100, and constant rows (rstd = eps^-1/2)"""
    x = _randn(M, 64, seed=seed)
    x[1::3] = x[1::3] + 100.0 * _randn(M, 1, seed=seed + 1)[1::3].sign()
    x[2::5] = _randn(M, 1, seed=seed + 2)[2::5].expand(-1, 64)
    return x


def _ffn_params(seed, g_weights=None, prefix=None):
    """(ln_g, ln_b, W1 (256, 64), b1, W2 (64, 256), b2).  Random: h = W1 xn + b1 spreads over +-40 (Swish saturated at both ends, and its
    neighbourhood of 0); or the shipped weights of one block"""
    if g_weights is not None:
        w = {k[len(prefix) + 1:]: v.float() for k, v in g_weights.items() if k.startswith(prefix + ".")}
        return (w["fn.norm.weight"], w["fn.norm.bias"], w["fn.fn.net.0.weight"], w["fn.fn.net.0.bias"], w["fn.fn.net.3.weight"],
                w["fn.fn.net.3.bias"])
    return (1.0 + 0.3 * _randn(64, seed=seed), 0.3 * _randn(64, seed=seed + 1), _randn(256, 64, seed=seed + 2, scale=1.5),
            _randn(256, seed=seed + 3, scale=2.0), _randn(64, 256, seed=seed + 4, scale=1 / 16), _randn(64, seed=seed + 5, scale=0.5))


def _ffn_masks(mode, M, seed1, seed2):
    """(thr, inv_keep, device counter, mask1 (M, 256), mask2 (M, 64)) as float64 scales: the library's hash on (m N + n) / 2"""
    counter = None
    if mode == "off":
        return 0, 1.0, None, torch.ones(M, 256, dtype=torch.float64), torch.ones(M, 64, dtype=torch.float64)
    if mode == "thr0":                               # dropout disabled by thr = 0 whatever inv_keep says
        return 0, 1.25, None, torch.ones(M, 256, dtype=torch.float64), torch.ones(M, 64, dtype=torch.float64)
    thr, inv = ops.drop_params(0.2)
    e1, e2 = seed1, seed2
    if mode == "dev":
        counter = torch.tensor([11], dtype=torch.int64, device=DEV)
        e1, e2 = _mix_seed(seed1, 11), _mix_seed(seed2, 11)
    m1 = _keep(e1, torch.arange(M * 256), thr).view(M, 256).double() * _f32(inv)
    m2 = _keep(e2, torch.arange(M * 64), thr).view(M, 64).double() * _f32(inv)
    return thr, inv, counter, m1, m2


def _ln_terms(x):
    """float64 LayerNorm statistics and the bounds of the kernel's (two threads per row, 32 sequential adds each and a shuffle):
    mean: 34 mean|x|; rstd (relative): half the variance's chain, rsqrtf, and the mean's error squared against var + eps"""
    x = x.double()
    mu = x.mean(1)
    var = x.var(1, unbiased=False)
    rstd = 1 / torch.sqrt(var + _f32(EPS))
    mabs = x.abs().mean(1)
    mean_err = 34 * mabs
    rstd_rel = 24 + 0.5 * (mean_err * U) ** 2 / (var + _f32(EPS)) / U
    return mu, rstd, mean_err, rstd_rel


def _ffn_fwd_ref(x, P, m1, m2):
    """float64 forward and the bounds (units of 2^-24) of xn, h, a and the branch 0.5 drop2(W2 a + b2)"""
    g, b, W1, b1, W2, b2 = (t.double().to(DEV) for t in P)
    x = x.double().to(DEV)
    m1, m2 = m1.to(DEV), m2.to(DEV)
    mu, rstd, mean_err, rstd_rel = _ln_terms(x)
    xhat = (x - mu[:, None]) * rstd[:, None]
    xn = xhat * g + b
    # xn = rna((x - mean) rstd g + b): rstd's error and four roundings on |xhat g|, the mean's error times rstd |g|, beta's add
    # (the rna itself is the tf32 term of the comparison, or TR |xn| where xn feeds the contraction)
    lim_xn = (rstd_rel[:, None] + 4) * (xhat * g).abs() + mean_err[:, None] * rstd[:, None] * g.abs() + 2 * b.abs()
    xn_abs = xn.abs()
    # h = xn W1^T + b1: xn's error and its rna (TR), W1's image rounded (TR), the 64-term chain and the bias add
    h = xn @ W1.t() + b1
    h_err = (lim_xn + TR * xn_abs) @ W1.abs().t() + (TR + 72) * (xn_abs @ W1.abs().t()) + b1.abs() + h.abs()
    sw, d1, d2, se, _ = _swish_terms(h)
    # a = rna(swish(h) mask): h's error through swish' (and half its square through swish'' <= 0.5), sigmoidf_ and two roundings
    a = sw * m1
    lim_a = m1 * (d1.abs() * h_err + 0.5 * U * h_err ** 2 + sw.abs() * (se + 2))
    # y = a W2^T + b2: a's error and its rna (TR), W2's image rounded (TR), the 256-term chain, the bias; the branch: alpha, mask (2)
    y = a @ W2.t() + b2
    y_err = (lim_a + TR * a.abs()) @ W2.abs().t() + (TR + 264) * (a.abs() @ W2.abs().t()) + b2.abs() + y.abs()
    br = 0.5 * y * m2
    lim_br = 0.5 * m2 * (y_err + 2 * y.abs())
    return dict(mu=mu, rstd=rstd, mean_err=mean_err, rstd_rel=rstd_rel, xhat=xhat, xn=xn, lim_xn=lim_xn, h=h, h_err=h_err, a=a, lim_a=lim_a,
                br=br, lim_br=lim_br)


def _rows_buf(t, ld, fill):
    """(M, 64) rows at leading dimension ld; the ld - 64 pad columns hold ``fill`` (NaN in an input shows a read, SENT in an output a write)"""
    M = t.shape[0]
    b = _buf(M * ld, fill)
    b[:M * ld].view(M, ld)[:, :64] = t.to(DEV)
    return b


def _ffn_M(spec):
    return {"sm": _nsm() * 64, "3sm+77": 3 * _nsm() * 64 + 77}.get(spec, spec)


FFN_M = [1, 63, 64, 65, 300, "sm", "3sm+77"]
FFN_MODES = ["host", "dev", "off", "thr0"]
S1, S2 = 0x0123456789ABCDEF, 0xF0E1D2C3B4A59687


def _ffn_fwd_case(M, mode, P, nm):
    ldx, ldo = 68, 66
    x = _ffn_x(M, 800)
    thr, inv, counter, m1, m2 = _ffn_masks(mode, M, S1, S2)
    if mode in ("host", "dev") and M >= 300:
        assert 0.7 < m1.ne(0).double().mean().item() < 0.9
    g, b, W1, b1, W2, b2 = (t.to(DEV) for t in P)
    xb = _rows_buf(x, ldx, NAN)
    out = _rows_buf(torch.full((M, 64), NAN), ldo, SENT)
    call("cmgan_ffn_fwd", xb, ldx, M, g, b, ops.packed_weight(W1, 0, 1, 64, 64, 1, 256), b1, ops.packed_weight(W2, 0, 1, 256, 256, 1, 64), b2,
         0.5, S1, S2, thr, inv, counter, out, ldo)
    _tail(out, M * ldo, "ffn_fwd out")
    o = out[:M * ldo].view(M, ldo).cpu()
    assert bool((o[:, 64:] == SENT).all()), "ffn_fwd wrote a guard column"
    R = _ffn_fwd_ref(x, P, m1, m2)
    x64 = x.double()
    ref_out = x64 + R["br"].cpu()
    # the branch out - x (exact in float64): its bound and the residual add's rounding of |out|
    _close(o[:, :64].double() - x64, R["br"].cpu(), R["lim_br"].cpu() + ref_out.abs(), 1, f"ffn_fwd branch {nm}")
    _close(o[:, :64], ref_out, R["lim_br"].cpu() + ref_out.abs(), 1, f"ffn_fwd out {nm}")


@pytest.mark.parametrize("mode", FFN_MODES)
@pytest.mark.parametrize("Ms", FFN_M)
def test_ffn_fwd(Ms, mode):
    M = _ffn_M(Ms)
    _ffn_fwd_case(M, mode, _ffn_params(810), f"M={M} {mode}")


def test_ffn_fwd_shipped(g_weights):
    M = _ffn_M("3sm+77")
    _ffn_fwd_case(M, "host", _ffn_params(0, g_weights, "TSCB_2.freq_conformer.ff1"), f"M={M} shipped TSCB_2.freq_conformer.ff1")


def _ffn_bwd_case(M, mode, res2_on, P, nm):
    ldx, lddz, lddo, ldr2, lddx = 68, 72, 76, 80, 84
    x = _ffn_x(M, 820)
    thr, inv, counter, m1, _ = _ffn_masks(mode, M, S1, S2)
    dz = tf32_rna((_randn(M, 64, seed=821, scale=0.5) * _keep(S2, torch.arange(M * 64), ops.drop_params(0.2)[0]).view(M, 64)))
    dout, res2 = _randn(M, 64, seed=822), _randn(M, 64, seed=823)
    g, b, W1, b1, W2, _ = (t.to(DEV) for t in P)
    xb, dzb, dob = _rows_buf(x, ldx, NAN), _rows_buf(dz, lddz, NAN), _rows_buf(dout, lddo, NAN)
    r2b = _rows_buf(res2, ldr2, NAN) if res2_on else None
    dx = _rows_buf(torch.full((M, 64), NAN), lddx, SENT)
    a_o, dh_o, xn_o, ws = _buf(M * 256), _buf(M * 256), _buf(M * 64), _buf(M * 66)
    dg0, db0 = _randn(64, seed=824), _randn(64, seed=825)
    dg, db = _buf(64, dg0), _buf(64, db0)
    call("cmgan_ffn_bwd", xb, ldx, dzb, lddz, dob, lddo, r2b, ldr2 if res2_on else 0, M, g, b, ops.packed_weight(W1, 0, 1, 64, 64, 1, 256), b1,
         ops.packed_weight(W2, 0, 256, 1, 64, 1, 256), ops.packed_weight(W1, 0, 64, 1, 256, 1, 64), S1, thr, inv, counter, dx, lddx, a_o, dh_o,
         xn_o, dg, db, ws)
    for bb, n, what in ((dx, M * lddx, "dx"), (a_o, M * 256, "a"), (dh_o, M * 256, "dh"), (xn_o, M * 64, "xn"), (ws, M * 66, "ws"),
                        (dg, 64, "dgamma"), (db, 64, "dbeta")):
        _tail(bb, n, f"ffn_bwd {what}")
    dxo = dx[:M * lddx].view(M, lddx).cpu()
    assert bool((dxo[:, 64:] == SENT).all()), "ffn_bwd wrote a guard column of dx"

    R = _ffn_fwd_ref(x, P, m1, torch.ones(M, 64, dtype=torch.float64))
    # float64 autograd of the module from its input to W2 a (b2, alpha and the second dropout are folded into dz)
    gl, bl = P[0].double().to(DEV).requires_grad_(), P[1].double().to(DEV).requires_grad_()
    xl = x.double().to(DEV).requires_grad_()
    xn = F.layer_norm(xl, (64,), gl, bl, eps=_f32(EPS))
    xn.retain_grad()
    h = xn @ P[2].double().to(DEV).t() + P[3].double().to(DEV)
    h.retain_grad()
    mask1 = m1.to(DEV)
    ((h * torch.sigmoid(h) * mask1) @ P[4].double().to(DEV).t()).backward(dz.double().to(DEV))
    with torch.no_grad():
        W1a, W2a = P[2].double().to(DEV).abs(), P[4].double().to(DEV).abs()
        dza = dz.double().to(DEV).abs()
        # dacc = dz W2 (64 terms): W2^T's image rounded (TR), the chain
        dacc = dz.double().to(DEV) @ P[4].double().to(DEV)
        dacc_err = (TR + 72) * (dza @ W2a)
        _, d1, d2, _, d1_err = _swish_terms(R["h"])
        # dh = rna(dacc swish'(h) mask): dacc's error, h's error through swish'' (and its square), swish''s own error, two roundings
        lim_dh = mask1 * (dacc.abs() * (d2.abs() * R["h_err"] + 0.5 * U * R["h_err"] ** 2 + d1_err) + dacc_err * d1.abs() +
                          2 * (dacc * d1).abs())
        dh_ref = h.grad
        # dLN = dh W1 on the row GEMM (256 terms): dh's error and its rna (TR), W1^T's image rounded (TR), the chain
        dln = xn.grad
        dln_err = (lim_dh + TR * dh_ref.abs()) @ W1a + (TR + 264) * (dh_ref.abs() @ W1a)
        # LayerNorm backward from the kernel's float32 stats: xhat's error (rstd's, three roundings, the mean's)
        xhat, rstd = R["xhat"], R["rstd"][:, None]
        xh_err = (R["rstd_rel"][:, None] + 3) * xhat.abs() + R["mean_err"][:, None] * rstd
        ga = gl.detach().abs()
        dga = (dln * gl.detach()).abs()
        A = rstd * (dga + dga.mean(1, keepdim=True) + xhat.abs() * (dga * xhat.abs()).mean(1, keepdim=True))
        Ae = rstd * (ga * dln_err + (ga * dln_err).mean(1, keepdim=True) + xhat.abs() * (ga * dln_err * xhat.abs()).mean(1, keepdim=True))
        m2v = (dln * gl.detach() * xhat).mean(1, keepdim=True).abs()
        Ax = rstd * (xh_err * m2v + xhat.abs() * (dga * xh_err).mean(1, keepdim=True))
        br = xl.grad
        # dx - dout - res2: the LayerNorm backward's float32 chain (16 A, as ln_bwd), dLN's error (Ae), xhat's (Ax), rstd's on the whole
        # branch, and the two residual adds
        radd = dout.double().to(DEV) + (res2.double().to(DEV) if res2_on else 0)
        lim_dx = 16 * A + Ae + Ax + R["rstd_rel"][:, None] * br.abs() + radd.abs() + (br + radd).abs()
    _close(dxo[:, :64].double() - dout.double() - (res2.double() if res2_on else 0), br.cpu(), lim_dx.cpu(), 1, f"ffn_bwd dx branch {nm}")
    _close_tf32(a_o[:M * 256], R["a"].reshape(-1), R["lim_a"].reshape(-1), f"ffn_bwd a {nm}")
    _close_tf32(dh_o[:M * 256], dh_ref.reshape(-1), lim_dh.reshape(-1), f"ffn_bwd dh {nm}")
    _close_tf32(xn_o[:M * 64], R["xn"].reshape(-1), R["lim_xn"].reshape(-1), f"ffn_bwd xn {nm}")
    st = ws[64 * M:66 * M].view(M, 2).cpu()
    _close(st[:, 0], R["mu"].cpu(), R["mean_err"].cpu(), 1, f"ffn_bwd stats mean {nm}")
    _close(st[:, 1], R["rstd"].cpu(), (R["rstd_rel"] * R["rstd"]).cpu(), 1, f"ffn_bwd stats rstd {nm}")
    # dgamma / dbeta on the prefill: ln_bwd's chain (8 rows per thread, 16 partials, one atomic per 128 rows, the prefill, xhat: as
    # test_ln_bwd), dLN's error and xhat's
    c = 8 + 16 + _cdiv(M, 128) + 1 + 3
    with torch.no_grad():
        lim_g = dg0.double().abs().to(DEV) + c * (dln.abs() * xhat.abs()).sum(0) + (dln_err * xhat.abs()).sum(0) + (dln.abs() * xh_err).sum(0)
        lim_b = db0.double().abs().to(DEV) + c * dln.abs().sum(0) + dln_err.sum(0)
    _close(dg[:64], dg0.double() + gl.grad.cpu(), lim_g.cpu(), 1, f"ffn_bwd dgamma {nm}")
    _close(db[:64], db0.double() + bl.grad.cpu(), lim_b.cpu(), 1, f"ffn_bwd dbeta {nm}")


@pytest.mark.parametrize("mode", FFN_MODES)
@pytest.mark.parametrize("Ms", FFN_M)
def test_ffn_bwd(Ms, mode):
    M = _ffn_M(Ms)
    res2_on = (FFN_M.index(Ms) + FFN_MODES.index(mode)) % 2 == 0
    _ffn_bwd_case(M, mode, res2_on, _ffn_params(830), f"M={M} {mode} res2={res2_on}")


def test_ffn_bwd_shipped(g_weights):
    M = _ffn_M("3sm+77")
    _ffn_bwd_case(M, "host", True, _ffn_params(0, g_weights, "TSCB_3.time_conformer.ff2"), f"M={M} shipped TSCB_3.time_conformer.ff2")


def test_ffn_m_zero():
    """M = 0: both entries return 0 and write nothing"""
    P = [t.to(DEV) for t in _ffn_params(840)]
    g, b, W1, b1, W2, b2 = P
    x, dz = _buf(64, 1.0), _buf(64, 1.0)
    out, dx, a_o, dh_o, xn_o, ws, dg, db = (_buf(0, SENT) for _ in range(8))
    call("cmgan_ffn_fwd", x, 64, 0, g, b, ops.packed_weight(W1, 0, 1, 64, 64, 1, 256), b1, ops.packed_weight(W2, 0, 1, 256, 256, 1, 64), b2,
         0.5, S1, S2, 0, 1.0, None, out, 64)
    call("cmgan_ffn_bwd", x, 64, dz, 64, x, 64, None, 0, 0, g, b, ops.packed_weight(W1, 0, 1, 64, 64, 1, 256), b1,
         ops.packed_weight(W2, 0, 256, 1, 64, 1, 256), ops.packed_weight(W1, 0, 64, 1, 256, 1, 64), S1, 0, 1.0, None, dx, 64, a_o, dh_o, xn_o,
         dg, db, ws)
    torch.cuda.synchronize()
    for t, nm in ((out, "out"), (dx, "dx"), (a_o, "a"), (dh_o, "dh"), (xn_o, "xn"), (ws, "ws"), (dg, "dgamma"), (db, "dbeta")):
        _tail(t, 0, f"ffn M = 0 {nm}")

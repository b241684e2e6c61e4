"""Float64 reference of attention (mmae_attention_forward / _backward and the fp32 tier's mmae_attention_f32_*), with an
error budget for every output element, input regimes, deliberately wrong references and a CPU emulation of the kernels'
arithmetic (tests/test_attention_oracle_host.py, tests/test_cuda_attention_float64.py).

Per head: S = scale q k^T, P = softmax(S), o = P v, lse = logsumexp(S); backward dv = P^T dO, dP = dO v^T,
Delta = rowsum(dO o), dS = P (dP - Delta), dq = scale dS k, dk = scale dS^T q.  The reference computes these in float64
on the very values the kernel is given (bf16, or fp32 for the fp32 tier), one chunk of heads at a time.

Budget derivation.  u_p is the rounding of the P / dS operands of the P V, P^T dO, dS k and dS^T q products (bf16:
u = 2^-8; fp32 tier: 0), u_s the rounding of the stored o, dq, dk, dv (bf16: u; fp32 tier: 0), e = 2^-24 the fp32 unit
roundoff.  Every product of two operands is exact in fp32; an fp32 sum of n terms is wrong by at most 2 n e times the
sum of their magnitudes (2 e per addition allows for tensor-core adders that truncate instead of rounding).
  * scores: sigma_ij = 2 (dh + 1) e sum_d |q_id k_jd| bounds the fp32 dot product (the + 1: the fp32 tier's q scale).
  * exp argument: the kernels form exp2(S log2e - m log2e) (or exp(S - m)); with M_i = max_j |S_ij| the roundings of the
    two products and the difference move the argument by at most 2 e (|S_ij| + M_i) natural units, and ex2.approx / expf
    add 4 e relative.  So the unnormalised p_ij has relative error at most
        eta_ij = scale sigma_ij + 2 e (|S_ij| + M_i) + 4 e  <=  eta_i = scale max_j sigma_ij + 4 e M_i + 4 e.
    A wrong max only shifts every p of the row by one factor, which the normalisation cancels.
  * o: P / l carries eta from p and eta from l, l's fp32 sum 2 Nk e, the fp32 P V sum 2 Nk e, the running-max rescale
    (acc and l multiplied by the same factor: 2 e per rescale, at most Nk of them) and 1 / l, acc / l: 4 e.
        F_i = 2 eta_i + (6 Nk + 4) e.
    P enters P V rounded to u_p, then the result is stored rounded to u_s:
        |o - o_ref|[i,d] <= ((u_p + F_i)(1 + u_s) + u_s) sum_j P_ij |v_jd|                                  (B_o)
  * lse = m scale + log(l): the score error reaches lse as a P-weighted mean (<= eta_i), l's sum 2 Nk e, logf and the
    two products / the sum 4 e of the magnitudes involved:
        |lse - lse_ref|_i <= eta_i + (2 Nk + 4) e (1 + M_i + |lse_i|)                                       (B_lse)
    No u term: l sums the unrounded p.
  * backward P is recomputed as exp2(S log2e - lse log2e) from the stored fp32 lse.  Its relative error is the score
    error, the argument rounding 2 e (|S_ij| + |lse_i|) - which grows with the size of the logits, not with the
    softmax's own values - the stored lse's own error B_lse and the exp: per row
        eta'_i = scale max_j sigma_ij + 2 e (M_i + |lse_i|) + 4 e + B_lse_i.
  * dv = P^T dO: P rounded to u_p, fp32 sum of Nq terms, store u_s:
        |dv - dv_ref|[j,d] <= sum_i ((u_p + eta'_i + 2 Nq e)(1 + u_s) + u_s) P_ij |dO_id|                   (B_dv)
  * Delta: the kernels form it from their own stored o in an fp32 dot of dh terms.  That o is sum_j P_ij (1 + d_ij) v_jd
    with one relative error |d_ij| <= (u_p + F_i)(1 + u_p) per weight, the same for every column d, plus the P V sum's
    2 Nk e per column, then rounded to u_s.  Summed against dO the weight errors give sum_j d_ij P_ij dP_ij, so
        E_i = (u_p + F_i)(1 + u_p) sum_j P_ij |dP_ij| + 2 Nk e sum_d |dO_id| (P |v|)_id
              + (u_s + 2 (dh + 1) e) sum_d |dO_id| (|o_id| + B_o[i,d]).
    dP is an fp32 dot: sigma'_ij = 2 (dh + 1) e sum_d |dO_id v_jd|.  dS_ij = P_ij (dP_ij - Delta_i) is then wrong by
    P's relative error, the difference's and product's roundings (3 e), its rounding to u_p, and P_ij (sigma'_ij + E_i)
    from its operands; dq = scale dS k adds the fp32 sum of Nk terms and the store:
        W_ij = P_ij (A_i |dP_ij - Delta_i| + C_i (sigma'_ij + E_i)),
        A_i = (u_p + eta'_i + (2 N + 4) e)(1 + u_s) + u_s,  C_i = (1 + u_p)(1 + u_s)(1 + eta'_i),  N = max(Nq, Nk)
        |dq - dq_ref| <= scale W |k|,   |dk - dk_ref| <= scale W^T |q|                                (B_dq, B_dk)
    At Nk = 1 the exact dq and dk are 0 (o = v_1, so dP = Delta); the E and sigma' terms still give a finite bound.
A correct kernel never exceeds any of these; an element over its budget is a finding.

Regimes (make_inputs): flat (randn * 0.5, near-uniform softmax), trained (scaled scores of standard deviation ~3), peaked
(each row has one key >= 20 above the rest, at key 0, in a middle 64-key chunk, at the first key of the last chunk or at
key Nk - 1: rows whose maximum arrives in a later chunk exercise the running-max rescale), ties (peaked, with those keys
duplicated in pairs across chunks), uniform (identical keys in a head: P = 1/Nk exactly), large_pos / large_neg (every
scaled score in [80, 120] / [-120, -80]: without the max subtraction exp overflows fp32 above 88.7, and falls below its
normal range under -87.3) and zero_do (trained, with whole dO rows exactly 0).

MUTATIONS (reference(..., mutate=...)) are wrong references that a test must tell apart from the kernels:
  "scale"          scale * (1 + 2^-5) everywhere;
  "drop_last_key"  key Nk - 1 left out (its dk, dv 0);
  "head_shift"     q of head h against k and v of head h + 1;
  "neighbour_keys" every sample's queries against the previous sample's keys;
  "no_rescale"     64-key chunks combined without the running-max rescale (backward from that forward's o and lse);
  "no_delta"       dS formed without Delta."""
import math

import torch

U = 2.0 ** -8                 # bf16 unit roundoff
E32 = 2.0 ** -24              # fp32 unit roundoff
LOG2E = 1.0 / math.log(2.0)
CHUNK = 64                    # keys per online-softmax chunk of the mma.sync kernels
TIERS = {"bf16": (U, U), "fp32": (0.0, 0.0)}           # (u_p, u_s)
TENSORS = ("o", "lse", "dq", "dk", "dv")
REGIMES = ("flat", "trained", "peaked", "ties", "uniform", "large_pos", "large_neg", "zero_do")
MUTATIONS = ("scale", "drop_last_key", "head_shift", "neighbour_keys", "no_rescale", "no_delta")
PEAK_GAP = 24.0               # scaled score of a peaked row's key above the base (the others: noise of std ~0.25)
LARGE_BASE = 90.0             # |scaled score| of the large regimes before the per-row / per-key factors and noise


def bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


# ---------------------------------------------------------------------------------------------------------------- inputs
def peak_keys(Nk):
    """the keys a peaked row may single out: 0, one in a middle 64-key chunk, the first of the last chunk, Nk - 1"""
    nch = (Nk + CHUNK - 1) // CHUNK
    mid = CHUNK * (nch // 2) + 17 if nch >= 3 else Nk // 2
    return sorted({0, min(mid, Nk - 1), CHUNK * ((Nk - 1) // CHUNK), Nk - 1})


def make_inputs(regime, B, H, Nq, Nk, dh, seed=0, tier="bf16"):
    """(q, k, v, do) as float32 [B, H, N, dh] on the CPU, bf16 values for the bf16 tier"""
    gen = torch.Generator().manual_seed(seed)
    scale = dh ** -0.5
    r = lambda n, s=1.0: torch.randn(B, H, n, dh, generator=gen) * s
    uni = lambda *shape: torch.rand(*shape, generator=gen)
    q, k, v, do = r(Nq, 0.5), r(Nk, 0.5), r(Nk, 0.5), r(Nq, 0.5)
    if regime in ("trained", "zero_do"):
        q, k = r(Nq, 3.0 ** 0.5), r(Nk, 3.0 ** 0.5)           # std(scale q.k) = 3
    elif regime in ("peaked", "ties"):
        pos = peak_keys(Nk)
        a = (PEAK_GAP / scale) ** 0.5
        q[..., :4] = 0.0
        k[..., :4] = 0.0
        for ax, p in enumerate(pos):
            k[:, :, p, ax] = a
        tgt = torch.arange(Nq) % len(pos)
        q[:, :, torch.arange(Nq), tgt] = a
        if regime == "ties" and Nk > 1:    # key Nk - 1 repeats key 0; the last chunk's first key the middle one
            k[:, :, Nk - 1] = k[:, :, 0]
            last = CHUNK * ((Nk - 1) // CHUNK)
            if len(pos) == 4 and last not in (0, Nk - 1):
                k[:, :, last] = k[:, :, pos[1]]
    elif regime == "uniform":
        k = r(1).expand(B, H, Nk, dh).clone()
        q = r(Nq, 1.0)
    elif regime in ("large_pos", "large_neg"):
        a0 = (LARGE_BASE / scale) ** 0.5
        sign = 1.0 if regime == "large_pos" else -1.0
        q, k = r(Nq, 1.2), r(Nk, 1.2)                         # std(scale q.k) over the other dims ~1.4
        q[..., 0] = sign * a0 * (1.0 + 0.15 * uni(B, H, Nq))
        k[..., 0] = a0 * (1.0 + 0.05 * uni(B, H, Nk))
    if regime == "zero_do":
        do[:, :, sorted({0, Nq // 2, Nq - 1})] = 0.0
    if tier == "bf16":
        q, k, v, do = (bf16(t) for t in (q, k, v, do))
    if regime == "ties":
        assert Nk == 1 or torch.equal(k[:, :, 0], k[:, :, Nk - 1])
    return q, k, v, do


# ------------------------------------------------------------------------------------------------------------ reference
def _gather(x, B, H, mutate, which):
    """[B*H, N, dh] operand of each head as the mutated reference reads it"""
    if mutate == "head_shift" and which in "kv":
        return x.reshape(B, H, *x.shape[1:]).roll(-1, 1).reshape(x.shape)
    if mutate == "neighbour_keys" and which == "k":
        return x.reshape(B, H, *x.shape[1:]).roll(1, 0).reshape(x.shape)
    return x


def _no_rescale(S):
    """weights exp(S_j - m_c) with m_c the running max at j's 64-key chunk, and the lse such a kernel stores"""
    Nk = S.shape[-1]
    m_run = torch.full(S.shape[:-1], -math.inf, dtype=S.dtype, device=S.device)
    w = torch.empty_like(S)
    for c0 in range(0, Nk, CHUNK):
        m_run = torch.maximum(m_run, S[..., c0:c0 + CHUNK].amax(-1))
        w[..., c0:c0 + CHUNK] = torch.exp(S[..., c0:c0 + CHUNK] - m_run[..., None])
    l = w.sum(-1)
    return w / l[..., None], m_run + torch.log(l)


def _heads(q, k, v, do, scale, tier, mutate, budget):
    """forward, backward and (budget=True) the budgets of G heads: [G, N, dh] float64 operands"""
    Nq, Nk, dh = q.shape[1], k.shape[1], q.shape[2]
    if mutate == "scale":
        scale = scale * (1.0 + 2.0 ** -5)
    kk, vv = (k[:, :-1], v[:, :-1]) if mutate == "drop_last_key" else (k, v)
    S = scale * (q @ kk.transpose(1, 2))
    if mutate == "no_rescale":
        Pf, lse = _no_rescale(S)
        P = torch.exp(S - lse[..., None])                     # what its backward recomputes from the stored lse
    else:
        lse = torch.logsumexp(S, -1)
        P = Pf = torch.exp(S - lse[..., None])
    o = Pf @ vv
    dv = P.transpose(1, 2) @ do
    dP = do @ vv.transpose(1, 2)
    delta = (do * o).sum(-1)
    if mutate == "no_delta":
        delta = torch.zeros_like(delta)
    dmd = dP - delta[..., None]
    dS = P * dmd
    dq, dk = scale * (dS @ kk), scale * (dS.transpose(1, 2) @ q)
    if mutate == "drop_last_key":
        pad = torch.zeros_like(k[:, :1])
        dk, dv = torch.cat([dk, pad], 1), torch.cat([dv, pad], 1)
    out = {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}
    if not budget:
        return out
    u_p, u_s = TIERS[tier]
    e = E32
    N = max(Nq, Nk)
    Sa = S.abs()
    M = Sa.amax(-1)
    sig = 2 * (dh + 1) * e * (q.abs() @ k.abs().transpose(1, 2))
    eta = scale * sig.amax(-1) + 4 * e * M + 4 * e
    F = 2 * eta + (6 * Nk + 4) * e
    b_o = (((u_p + F) * (1 + u_s) + u_s)[..., None]) * (P @ v.abs())
    b_lse = eta + (2 * Nk + 4) * e * (1 + M + lse.abs())
    eta_b = scale * sig.amax(-1) + 2 * e * (M + lse.abs()) + 4 * e + b_lse
    c_dv = (u_p + eta_b + 2 * Nq * e) * (1 + u_s) + u_s
    b_dv = P.transpose(1, 2) @ (c_dv[..., None] * do.abs())
    pv = P @ v.abs()
    E = ((u_p + F) * (1 + u_p)) * (P * dP.abs()).sum(-1) + 2 * Nk * e * (do.abs() * pv).sum(-1) + \
        (u_s + 2 * (dh + 1) * e) * (do.abs() * (o.abs() + b_o)).sum(-1)
    sig_p = 2 * (dh + 1) * e * (do.abs() @ v.abs().transpose(1, 2))
    A = (u_p + eta_b + (2 * N + 4) * e) * (1 + u_s) + u_s
    C = (1 + u_p) * (1 + u_s) * (1 + eta_b)
    W = P * (A[..., None] * dmd.abs() + C[..., None] * (sig_p + E[..., None]))
    out.update(b_o=b_o, b_lse=b_lse, b_dv=b_dv, b_dq=scale * (W @ k.abs()), b_dk=scale * (W.transpose(1, 2) @ q.abs()))
    return out


def head_chunks(B, H, Nq, Nk, max_elems=1 << 24):
    """ranges of flattened (b, h) heads whose [Nq, Nk] float64 score matrices hold at most max_elems elements"""
    n = max(1, max_elems // max(1, Nq * Nk))
    return [(g, min(g + n, B * H)) for g in range(0, B * H, n)]


def reference(q, k, v, do, scale, tier="bf16", mutate=None, budget=True, heads=None):
    """float64 o, lse, dq, dk, dv (and with budget=True their budgets b_<name>) of the heads [g0, g1) of [B, H, N, dh]
    operands (any float dtype, any device): [g1 - g0, ...] tensors.  heads=None: all heads."""
    B, H = q.shape[:2]
    g0, g1 = heads if heads is not None else (0, B * H)
    flat = lambda x: x.reshape(B * H, *x.shape[2:])
    qf, kf, vf, df = flat(q), _gather(flat(k), B, H, mutate, "k"), _gather(flat(v), B, H, mutate, "v"), flat(do)
    d = lambda x: x[g0:g1].double()
    return _heads(d(qf), d(kf), d(vf), d(df), scale, tier, mutate, budget and mutate is None)


def ratio(got, want, bud):
    """elementwise |got - want| / budget: 0 where both are 0, inf where the budget is 0 and the error not (or NaN)"""
    err = (got.double() - want).abs()
    r = err / bud
    r = torch.where(err == 0, torch.zeros_like(r), r)
    return torch.nan_to_num(r, nan=math.inf)


# ------------------------------------------------------------------------------------------------------------ emulation
def emulate(q, k, v, do, scale, tier="bf16"):
    """The kernels' arithmetic in fp32 on the CPU for [B, H, N, dh] operands: dict of o, lse, dq, dk, dv ([B*H, ...]).

    bf16 tier (attention.cu's mma.sync kernels): fp32 scores of the bf16 operands; 64-key chunks with a running max,
    p = exp2(S log2e - m log2e) on the fp32 argument, P rounded to bf16 for P V, the fp32 row sum of the unrounded p,
    acc and l rescaled by exp2((m_old - m) scale log2e); o stored bf16, lse = m scale + log(l).  Backward: P recomputed
    from the fp32 lse, Delta from the bf16 o, dS = bf16(P (dP - Delta)), dv = bf16(bf16(P)^T dO), dq / dk stored bf16.
    fp32 tier (fp32_ops.cu): q pre-scaled in fp32, the same chunked online softmax with exp, no bf16 roundings."""
    B, H = q.shape[:2]
    f = lambda x: x.reshape(B * H, *x.shape[2:]).float()
    qf, kf, vf, df = f(q), f(k), f(v), f(do)
    Nk = kf.shape[1]
    rb = bf16 if tier == "bf16" else (lambda x: x)
    one = lambda x: torch.tensor(x, dtype=torch.float32)
    sc = one(scale)
    if tier == "bf16":
        s = qf @ kf.transpose(1, 2)
        sl2 = one(scale * LOG2E)
        arg = lambda a, m: torch.exp2(a * sl2 - m * sl2)
    else:
        s = (qf * sc) @ kf.transpose(1, 2)
        arg = lambda a, m: torch.exp(a - m)
    m_run = torch.full(s.shape[:-1], -math.inf)
    l = torch.zeros(s.shape[:-1])
    acc = torch.zeros(qf.shape[:2] + vf.shape[2:])
    for c0 in range(0, Nk, CHUNK):
        blk = s[..., c0:c0 + CHUNK]
        mx = torch.maximum(m_run, blk.amax(-1))
        alpha = torch.where(torch.isinf(m_run), torch.zeros_like(mx), arg(m_run, mx))
        p = arg(blk, mx[..., None])
        l = l * alpha + p.sum(-1)
        acc = acc * alpha[..., None] + rb(p) @ vf[:, c0:c0 + CHUNK]
        m_run = mx
    o = rb(acc * (1.0 / l)[..., None])
    if tier == "bf16":
        lse = m_run * sc + torch.log(l)
        P = torch.exp2(s * sl2 - (lse * one(LOG2E))[..., None])
    else:
        lse = m_run + torch.log(l)
        P = torch.exp(s - lse[..., None])
    delta = (df * o).sum(-1)
    dS = rb(P * (df @ vf.transpose(1, 2) - delta[..., None]))
    dv = rb(rb(P).transpose(1, 2) @ df)
    dq = rb((dS @ kf) * sc)
    dk = rb((dS.transpose(1, 2) @ qf) * sc)
    return {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}

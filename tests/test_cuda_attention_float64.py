"""GPU: every attention kernel family against the float64 reference of tests/attention_oracle.py, element by element.

MMAE_ATTN_TC = 0 runs the mma.sync forward (64-key chunks, online softmax) and, up to 256 keys, the fused backward, above
that delta + dQ + dK/dV; 7 runs the wgmma forward (one 128- or 256-key tile, mma.sync above 256 keys) and the wgmma
backward behind the delta kernel.  The fp32 tier (mmae_attention_f32_*) runs at head_dim 32.  Between them these reach
every attention kernel.  Each case runs in several input regimes (attention_oracle.REGIMES: peaked rows whose maximum
arrives in a later chunk, ties, identical keys, scaled scores of +-80..120, zero dO rows) and every element of o, lse, dq,
dk and dv must lie within its budget (derived in attention_oracle's docstring); the worst err / budget per (family,
regime, tensor) is printed.  Wrong references (a 2^-5 scale error, the last key dropped, the neighbouring head's or
sample's keys, chunks combined without the running-max rescale, dS without Delta) must miss the kernels' outputs by at
least 10x.

Before each call o, lse, dq, dk, dv and the delta workspace are NaN, so an element never written fails its budget; the
columns right of each strided view and a tail past B*H*Nq of lse and delta hold a sentinel that must survive.  The other
MMAE_ATTN_TC masks are pinned bit for bit to the two families on the key ranges where they select them, and two launches
give the same bits."""
import collections
import zlib

import pytest
import torch

import attention_oracle as AO
from multimae_b200 import _lib as L

pytestmark = pytest.mark.gpu

SENT = 7.0                 # margin sentinel of the bf16 / fp32 output buffers
TAIL = 64                  # lse / delta elements past B*H*Nq that must stay untouched
MISS = 10.0
WORST = collections.defaultdict(float)      # (family, regime, tensor) -> worst err / budget

# name: (B, H, Nq, Nk, dh, layout, regimes).  layout "self": q, k, v (and dq, dk, dv) are column views of one qkv (dqkv)
# buffer; "cross": q alone, k, v views of one kv buffer.  pad: extra columns right of every buffer (ld > its views)
ALL, BENCH = AO.REGIMES, ("flat", "trained")
CASES = {
    # the benchmark's shapes (MultiMAE-B bs 128 pre-training; cfg5 at 448^2; fine-tuning cls / 512^2 / segmenter)
    "encoder": (128, 12, 99, 99, 64, "self", BENCH),
    "dec_cross": (128, 8, 196, 99, 32, "cross", BENCH),
    "dec_self": (128, 8, 196, 196, 32, "self", BENCH),
    "cfg5_enc": (32, 12, 393, 393, 64, "self", ("trained",)),
    "cfg5_dec": (32, 8, 784, 784, 32, "self", ("trained",)),
    "ft_cls": (32, 12, 197, 197, 64, "self", ("trained",)),
    "ft_512": (4, 12, 1025, 1025, 64, "self", ("trained",)),
    "segmenter": (4, 12, 1175, 1175, 64, "self", ("trained", "peaked")),
    # edges in Nk around the 16-key groups, the 64-key chunks, the 128 / 256-key wgmma tiles and the fused backward's 256
    "nk1": (2, 3, 17, 1, 64, "cross", ALL),
    "nk5": (2, 2, 63, 5, 32, "cross", ALL),
    "nk16": (2, 2, 65, 16, 64, "cross", ALL),
    "nk17": (2, 2, 64, 17, 32, "cross", ALL),
    "nk63": (2, 2, 17, 63, 64, "cross", ALL),
    "nk64": (2, 2, 1, 64, 32, "cross", ALL),
    "nk65": (2, 2, 65, 65, 64, "self", ALL),
    "nk127": (2, 2, 63, 127, 32, "cross", ALL),
    "nk128": (2, 3, 128, 128, 64, "self", ALL),
    "nk129": (1, 4, 200, 129, 32, "cross", ALL),
    "nk255": (2, 2, 200, 255, 32, "cross", ALL),
    "nk256": (2, 3, 256, 256, 64, "self", ALL),
    "nk257": (1, 2, 257, 257, 32, "self", ALL),
    "nk257_cross": (2, 2, 150, 257, 64, "cross", ALL),
    "nq1_nk200": (3, 2, 1, 200, 64, "cross", ALL),
    # the shapes the earlier fp32-reference tests ran
    "enc_b3": (3, 12, 99, 99, 64, "self", BENCH),
    "enc_h16": (2, 16, 99, 99, 64, "self", BENCH),
    "dec_cross_b2": (2, 8, 196, 99, 32, "cross", BENCH),
    "dec_self_b2": (2, 8, 196, 196, 32, "self", BENCH),
    "dec_self_b5": (5, 8, 196, 196, 32, "self", BENCH),
    "n256_b1": (1, 2, 256, 256, 64, "self", BENCH),
    "n393": (1, 2, 393, 393, 64, "self", BENCH),
    "q130_k70": (1, 2, 130, 70, 32, "cross", BENCH),
    "q17_k5": (2, 1, 17, 5, 64, "cross", BENCH),
    "q100_k33": (1, 2, 100, 33, 64, "cross", BENCH),
    "q40_k7": (2, 3, 40, 7, 64, "cross", BENCH),
    "q5_k2": (3, 2, 5, 2, 32, "cross", BENCH),
    "n15": (2, 4, 15, 15, 32, "self", BENCH),
    "q70_k16": (1, 2, 70, 16, 64, "cross", BENCH),
}
PADDED = {"nk5": 8, "nk17": 24, "nk65": 16, "nk127": 8}     # ld = view width + pad


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    yield torch.device("cuda:0")
    print("\nworst err / budget per (family, regime, tensor):")
    for key in sorted(WORST):
        print("  %-6s %-10s %-4s %.3f" % (*key, WORST[key]))


@pytest.fixture
def tc():
    yield lambda mask: L.check(L.lib().mmae_attention_set_tc(mask), "mmae_attention_set_tc")
    L.lib().mmae_attention_set_tc(-1)


# ------------------------------------------------------------------------------------------------------------- buffers
def _rows(x):
    """[B, H, N, dh] -> [B*N, H*dh] (the projection buffers' row layout)"""
    B, H, N, dh = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * N, H * dh)


def _heads(x, B, H, N, dh):
    """[B*N, >= H*dh] view -> [B*H, N, dh] copy"""
    return x[:, :H * dh].reshape(B, N, H, dh).permute(0, 2, 1, 3).reshape(B * H, N, dh)


class Bufs:
    """device inputs and NaN-filled outputs of one call, in the case's layout, with sentinel margins"""

    def __init__(self, inputs, layout, pad, dtype, dev):
        q, k, v, do = inputs
        B, H, Nq, dh = q.shape
        Nk, D = k.shape[2], H * dh
        self.shape = (B, H, Nq, Nk, dh)
        full = lambda rows, cols: torch.full((rows, cols + pad), SENT, dtype=dtype, device=dev)
        if layout == "self":
            assert Nq == Nk
            qkv = full(B * Nq, 3 * D)
            for i, t in enumerate((q, k, v)):
                qkv[:, i * D:(i + 1) * D] = _rows(t).to(dev, dtype)
            self.q, self.k, self.v = (qkv[:, i * D:(i + 1) * D] for i in range(3))
            self.grad_bufs = [full(B * Nq, 3 * D)]
            self.dq, self.dk, self.dv = (self.grad_bufs[0][:, i * D:(i + 1) * D] for i in range(3))
        else:
            qb, kv = full(B * Nq, D), full(B * Nk, 2 * D)
            qb[:, :D] = _rows(q).to(dev, dtype)
            kv[:, :D], kv[:, D:2 * D] = _rows(k).to(dev, dtype), _rows(v).to(dev, dtype)
            self.q, self.k, self.v = qb[:, :D], kv[:, :D], kv[:, D:2 * D]
            self.grad_bufs = [full(B * Nq, D), full(B * Nk, 2 * D)]
            self.dq, self.dk, self.dv = self.grad_bufs[0][:, :D], self.grad_bufs[1][:, :D], self.grad_bufs[1][:, D:2 * D]
        dob = full(B * Nq, D)
        dob[:, :D] = _rows(do).to(dev, dtype)
        self.do = dob[:, :D]
        self.o_buf = full(B * Nq, D + 8)          # ldo > H * dh in every case
        self.o = self.o_buf[:, :D]
        n = B * H * Nq
        self.lse_buf = torch.full((n + TAIL,), SENT, dtype=torch.float32, device=dev)
        self.delta_buf = torch.full((n + TAIL,), SENT, dtype=torch.float32, device=dev)
        self.lse, self.delta = self.lse_buf[:n], self.delta_buf[:n]

    def nan_fwd(self):
        self.o.fill_(float("nan"))
        self.lse.fill_(float("nan"))

    def nan_bwd(self):
        for t in (self.dq, self.dk, self.dv, self.delta):
            t.fill_(float("nan"))

    def check_margins(self):
        D = self.q.shape[1]
        n = self.lse.numel()
        assert bool((self.o_buf[:, D:] == SENT).all()), "o margin written"
        assert bool((self.lse_buf[n:] == SENT).all()) and bool((self.delta_buf[n:] == SENT).all()), "lse / delta tail"
        for g, views in zip(self.grad_bufs, ([self.dq, self.dk, self.dv],) if len(self.grad_bufs) == 1 else
                            ([self.dq], [self.dk, self.dv])):
            assert bool((g[:, len(views) * D:] == SENT).all()), "gradient margin written"

    def outputs(self):
        B, H, Nq, Nk, dh = self.shape
        return {"o": _heads(self.o, B, H, Nq, dh), "lse": self.lse.reshape(B * H, Nq), "dq": _heads(self.dq, B, H, Nq, dh),
                "dk": _heads(self.dk, B, H, Nk, dh), "dv": _heads(self.dv, B, H, Nk, dh)}


def _call_bf16(b, scale):
    B, H, Nq, Nk, dh = b.shape
    lib, st = L.lib(), L.current_stream()
    b.nan_fwd()
    L.check(lib.mmae_attention_forward(b.q.data_ptr(), b.q.stride(0), b.k.data_ptr(), b.k.stride(0), b.v.data_ptr(),
                                       b.v.stride(0), b.o.data_ptr(), b.o.stride(0), b.lse.data_ptr(), B, H, Nq, Nk, dh,
                                       scale, 0.0, None, st), "mmae_attention_forward")
    _call_bf16_bwd(b, scale)


def _call_bf16_bwd(b, scale):
    B, H, Nq, Nk, dh = b.shape
    b.nan_bwd()
    L.check(L.lib().mmae_attention_backward(b.q.data_ptr(), b.q.stride(0), b.k.data_ptr(), b.k.stride(0), b.v.data_ptr(),
                                            b.v.stride(0), b.o.data_ptr(), b.o.stride(0), b.do.data_ptr(), b.do.stride(0),
                                            b.lse.data_ptr(), b.delta.data_ptr(), b.dq.data_ptr(), b.dq.stride(0),
                                            b.dk.data_ptr(), b.dk.stride(0), b.dv.data_ptr(), b.dv.stride(0), B, H, Nq, Nk,
                                            dh, scale, 0.0, None, L.current_stream()), "mmae_attention_backward")


def _call_f32(b, scale):
    B, H, Nq, Nk, dh = b.shape
    lib, st = L.lib(), L.current_stream()
    b.nan_fwd()
    L.check(lib.mmae_attention_f32_forward(b.q.data_ptr(), b.q.stride(0), b.k.data_ptr(), b.k.stride(0), b.v.data_ptr(),
                                           b.v.stride(0), b.o.data_ptr(), b.o.stride(0), b.lse.data_ptr(), B, H, Nq, Nk, dh,
                                           scale, st), "mmae_attention_f32_forward")
    b.nan_bwd()
    L.check(lib.mmae_attention_f32_backward(b.q.data_ptr(), b.q.stride(0), b.k.data_ptr(), b.k.stride(0), b.v.data_ptr(),
                                            b.v.stride(0), b.o.data_ptr(), b.o.stride(0), b.do.data_ptr(), b.do.stride(0),
                                            b.lse.data_ptr(), b.delta.data_ptr(), b.dq.data_ptr(), b.dq.stride(0),
                                            b.dk.data_ptr(), b.dk.stride(0), b.dv.data_ptr(), b.dv.stride(0), B, H, Nq, Nk,
                                            dh, scale, st), "mmae_attention_f32_backward")


# ------------------------------------------------------------------------------------------------------------ checking
def _against(runs, inputs, scale, tier, mutate=None):
    """worst |got - ref| / budget of each run's tensors against the exact reference (mutate=None, budgets of its own) or
    the mutated one (budgets of the exact reference): {run: {tensor: (ratio, (b, h, row, col))}}"""
    q, k, v, do = (t.to(runs[next(iter(runs))]["o"].device) for t in inputs)
    B, H, Nq, Nk = q.shape[0], q.shape[1], q.shape[2], k.shape[2]
    worst = {name: {t: (0.0, None) for t in AO.TENSORS} for name in runs}
    for g0, g1 in AO.head_chunks(B, H, Nq, Nk):
        ref = AO.reference(q, k, v, do, scale, tier=tier, heads=(g0, g1))
        want = ref if mutate is None else AO.reference(q, k, v, do, scale, tier=tier, mutate=mutate, budget=False,
                                                       heads=(g0, g1))
        for name, got in runs.items():
            for t in AO.TENSORS:
                r = AO.ratio(got[t][g0:g1], want[t], ref["b_" + t])
                i = int(r.argmax())
                val = float(r.flatten()[i])
                if val > worst[name][t][0] or worst[name][t][1] is None:
                    idx = list(torch.unravel_index(torch.tensor(i), r.shape))
                    g = g0 + int(idx[0])
                    where = (g // H, g % H) + tuple(int(x) for x in idx[1:])
                    worst[name][t] = (max(val, worst[name][t][0]), where)
        del ref, want
    return worst


def _assert_within(worst, regime, label):
    bad = []
    for name, per in worst.items():
        for t, (r, where) in per.items():
            WORST[(name, regime, t)] = max(WORST[(name, regime, t)], r)
            if not r <= 1.0:
                bad.append((name, t, round(r, 3), "(b, h, row[, col])", where))
    assert not bad, (label, regime, bad)


def _mutations_miss(runs, inputs, scale, tier, B, H, Nk):
    for m in AO.MUTATIONS:
        if {"drop_last_key": Nk == 1, "head_shift": H == 1, "neighbour_keys": B == 1,
                "no_rescale": Nk <= AO.CHUNK}.get(m, False):
            continue
        worst = _against(runs, inputs, scale, tier, mutate=m)
        for name, per in worst.items():
            assert max(r for r, _ in per.values()) >= MISS, (m, name, {t: round(r, 2) for t, (r, _) in per.items()})


FAMILIES = {"tc0": 0, "tc7": 7}


@pytest.mark.parametrize("case", list(CASES))
def test_bf16_kernels_within_float64_budget(dev, tc, case):
    B, H, Nq, Nk, dh, layout, regimes = CASES[case]
    scale = dh ** -0.5
    for regime in regimes:
        inputs = AO.make_inputs(regime, B, H, Nq, Nk, dh, seed=zlib.crc32((case + regime).encode()) % 1000)
        runs = {}
        for fam, mask in FAMILIES.items():
            tc(mask)
            b = Bufs(inputs, layout, PADDED.get(case, 0), torch.bfloat16, dev)
            _call_bf16(b, scale)
            torch.cuda.synchronize()
            b.check_margins()
            runs[fam] = b.outputs()
        _assert_within(_against(runs, inputs, scale, "bf16"), regime, case)
        if regime == "trained" and B * H * Nq * Nk <= 1 << 22:
            _mutations_miss(runs, inputs, scale, "bf16", B, H, Nk)


F32_CASES = {          # B, H, Nq, Nk, layout, regimes (head_dim 32)
    "q16_k13": (3, 4, 16, 13, "cross", ALL),
    "dec_cross": (2, 8, 196, 99, "cross", ALL),
    "dec_self": (2, 8, 196, 196, "self", ALL),
    "q196_k196": (2, 8, 196, 196, "cross", ALL),
    "q130_k70": (1, 2, 130, 70, "cross", ALL),
    "nk1": (2, 2, 33, 1, "cross", ALL),
    "nk257": (1, 3, 70, 257, "cross", ALL),
    "dec_self_b32": (32, 8, 196, 196, "self", ("trained",)),
}
F32_PADDED = {"nk1": 4, "nk257": 12}


@pytest.mark.parametrize("case", list(F32_CASES))
def test_fp32_tier_within_float64_budget(dev, case):
    B, H, Nq, Nk, layout, regimes = F32_CASES[case]
    dh, scale = 32, 32 ** -0.5
    for regime in regimes:
        inputs = AO.make_inputs(regime, B, H, Nq, Nk, dh, seed=zlib.crc32((case + regime).encode()) % 1000, tier="fp32")
        b = Bufs(inputs, layout, F32_PADDED.get(case, 0), torch.float32, dev)
        _call_f32(b, scale)
        torch.cuda.synchronize()
        b.check_margins()
        runs = {"fp32": b.outputs()}
        _assert_within(_against(runs, inputs, scale, "fp32"), regime, case)
        if regime == "trained" and B * H * Nq * Nk <= 1 << 22:
            _mutations_miss(runs, inputs, scale, "fp32", B, H, Nk)


# --------------------------------------------------------------------------------------------------- dispatch, repeats
@pytest.mark.parametrize("Nk", [1, 64, 128, 129, 200, 256, 257, 300])
@pytest.mark.parametrize("dh", [32, 64])
def test_switch_masks_pinned_to_the_two_families(dev, tc, Nk, dh):
    """forward: bit 1 alone is tc 7 up to 128 keys, tc 0 above; bits 2, 8, 32, 128 are tc 7 for 129..256 keys, tc 0
    elsewhere.  Backward: bit 64 alone is bit 4 alone (the wgmma backward), masks without either are tc 0.  Bit 16 changes
    nothing.  Compared: o, lse, dq, dk, dv and the delta workspace, bit for bit."""
    B, H, Nq = 2, 3, 70
    scale = dh ** -0.5
    inputs = AO.make_inputs("trained", B, H, Nq, Nk, dh, seed=Nk)

    def fwd(mask):
        tc(mask)
        b = Bufs(inputs, "cross", 0, torch.bfloat16, dev)
        _call_bf16(b, scale)
        return b

    def bwd(mask, base):       # gradients and the delta workspace (NaN where a kernel leaves it alone), as bits
        tc(mask)
        _call_bf16_bwd(base, scale)
        return [t.clone().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)
                for t in (base.dq, base.dk, base.dv, base.delta)]

    ref = {m: fwd(m) for m in (0, 7)}
    for mask in (1, 2, 8, 32, 128, 16, 7 | 16, 1 | 16):
        wg = (mask & 1 and Nk <= 128) or (mask & (2 | 8 | 32 | 128) and 128 < Nk <= 256)
        got = fwd(mask)
        want = ref[7 if wg else 0]
        assert torch.equal(got.o, want.o) and torch.equal(got.lse, want.lse), (mask, Nk, dh)
    base = ref[0]
    g0, g4 = bwd(0, base), bwd(4, base)
    for mask, want in ((64, g4), (4 | 16, g4), (7, g4), (1, g0), (2, g0), (8, g0), (16, g0), (32, g0), (128, g0),
                       (1 | 2 | 8 | 32 | 128, g0)):
        for a, w in zip(bwd(mask, base), want):
            assert torch.equal(a, w), (mask, Nk, dh)
    # the two families are different kernels.  The forwards round differently; the backwards accumulate in the same
    # order and can agree to the bit, but up to 256 keys the fused one forms Delta itself and leaves the workspace alone
    if 1 < Nk <= 256:
        assert not torch.equal(ref[0].o, ref[7].o), (Nk, dh)
    if Nk <= 256:
        assert not torch.equal(g0[3], g4[3]), (Nk, dh)


@pytest.mark.parametrize("case", [(16, 12, 99, 99, 64), (16, 8, 196, 196, 32), (2, 4, 300, 300, 64)])
@pytest.mark.parametrize("mask", [0, 7])
def test_bitwise_repeatable(dev, tc, case, mask):
    """every o / lse / dq / dk / dv element is written by one thread, without atomics: two launches, equal bits"""
    B, H, Nq, Nk, dh = case
    scale = dh ** -0.5
    tc(mask)
    inputs = AO.make_inputs("trained", B, H, Nq, Nk, dh)
    outs = []
    for _ in range(2):
        b = Bufs(inputs, "self", 0, torch.bfloat16, dev)
        _call_bf16(b, scale)
        outs.append(b.outputs())
    for t in AO.TENSORS:
        assert torch.equal(outs[0][t], outs[1][t]), (t, case, mask)

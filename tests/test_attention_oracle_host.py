"""CPU: the attention budgets of tests/attention_oracle.py before any GPU run.  In every input regime and at shapes on both
sides of the 64-key chunk, the fp32 emulation of the kernels' arithmetic stays within every element's budget (not too
tight), and every wrong reference misses the exact one by at least 10x its budget (tight enough) - for the bf16 kernels
and for the fp32 tier."""
import math

import pytest
import torch

import attention_oracle as AO

# B, H, Nq, Nk, dh: one key, a ragged single chunk, a full chunk, and three chunks with a ragged last one (the fp32
# tier: the head_dim 32 ones)
SHAPES = [(2, 2, 17, 1, 32), (2, 2, 33, 5, 64), (2, 2, 65, 64, 32), (2, 2, 64, 150, 64), (2, 2, 5, 200, 32)]
MISS = 10.0
# (mutation, regime) -> the least miss there, where a regime leaves a mutation (almost) nothing to change:
#  * identical keys give every key the same score, so the running max never grows past the first chunk and skipping its
#    rescale changes nothing;
#  * in the flat regime o is an average of many v rows, |o| ~ |v| / sqrt(Nk), so Delta = dO . o is small next to dP and
#    dropping it moves dq / dk by a few budgets only.
WEAK = {("no_rescale", "uniform"): 0.0, ("no_delta", "flat"): 3.0}


def _worst(got, ref):
    return {n: float(AO.ratio(got[n], ref[n], ref["b_" + n]).max()) for n in AO.TENSORS}


def _applies(mutate, B, H, Nk):
    return {"drop_last_key": Nk > 1, "head_shift": H > 1, "neighbour_keys": B > 1, "no_rescale": Nk > AO.CHUNK}.get(
        mutate, True)


@pytest.mark.parametrize("regime", AO.REGIMES)
@pytest.mark.parametrize("tier,shape", [("bf16", s) for s in SHAPES] + [("fp32", s) for s in SHAPES if s[4] == 32],
                         ids=lambda x: "x".join(map(str, x)) if isinstance(x, tuple) else x)
def test_emulation_within_budget_and_mutations_miss(tier, shape, regime):
    B, H, Nq, Nk, dh = shape
    scale = dh ** -0.5
    q, k, v, do = AO.make_inputs(regime, B, H, Nq, Nk, dh, seed=Nq + Nk, tier=tier)
    ref = AO.reference(q, k, v, do, scale, tier=tier)
    worst = _worst(AO.emulate(q, k, v, do, scale, tier=tier), ref)
    assert max(worst.values()) <= 1.0, worst
    for m in AO.MUTATIONS:
        if not _applies(m, B, H, Nk):
            continue
        wrong = AO.reference(q, k, v, do, scale, tier=tier, mutate=m, budget=False)
        miss = _worst(wrong, ref)
        assert max(miss.values()) >= WEAK.get((m, regime), MISS), (m, miss)


@pytest.mark.parametrize("regime", AO.REGIMES)
def test_regimes_are_what_they_claim(regime):
    B, H, Nq, Nk, dh = 2, 3, 70, 200, 64
    q, k, v, do = AO.make_inputs(regime, B, H, Nq, Nk, dh)
    S = (q.double() @ k.double().transpose(-1, -2)) * dh ** -0.5
    top = S.topk(2, -1).values
    if regime == "trained":
        assert 2.5 < float(S.std()) < 3.5
    elif regime == "peaked":
        peak = S.argmax(-1)
        assert bool((top[..., 0] - top[..., 1] >= 20).all())
        assert set(peak.flatten().tolist()) == set(AO.peak_keys(Nk))          # the max arrives in every chunk position
    elif regime == "ties":
        assert bool((S.amax(-1)[..., ::4] == S[..., 0][..., ::4]).all())
        assert bool((top[..., 0] == top[..., 1]).any(-1).all())
    elif regime == "uniform":
        P = torch.softmax(S, -1)
        assert bool((P == P[..., :1]).all())
    elif regime in ("large_pos", "large_neg"):
        lo, hi = (80, 120) if regime == "large_pos" else (-120, -80)
        assert float(S.min()) >= lo and float(S.max()) <= hi
        ex = torch.exp(S.float())          # without the max subtraction: fp32 overflow / below the normal range
        assert math.isinf(float(ex.max())) if regime == "large_pos" else float(ex.min()) < torch.finfo(torch.float32).tiny
    elif regime == "zero_do":
        assert bool((do[:, :, 0] == 0).all() and (do[:, :, Nq - 1] == 0).all())

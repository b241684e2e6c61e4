"""GPU: the input / output side of a pre-training step through the C ABI, entry point by entry point, against float64.

1. mmae_embed_*, mmae_ctxproj_*, mmae_dectail_*: bit-exact.  Every input is dyadic (k / 8 or k / 16, |k| <= 8), so every
   product is a multiple of 2^-q and every sum the kernels form - in any order, split-K or atomics - stays below 2^(23-q)
   and is exact in fp32; bf16 casts of the inputs are exact and a bf16 output is the round-to-nearest-even of an exact
   value.  Each test asserts these premises on its reference before comparing with torch.equal.  The one inexact sum, the
   class-embedding scatter of bf16-rounded dA values, is held to 1e-6 of the sum of its terms' magnitudes per table row.
2. mmae_dechead_* against a float64 reference that rounds to bf16 wherever the kernels store bf16 (values and gradient
   operands, both GELU modes, the attention backward's row term from the stored bf16 output).  What it does NOT mirror:
     * attention's bf16 P (forward, and P / dS in backward): one bf16 rounding, relative u = 2^-8, per element;
     * __expf, fp32 accumulation order, LayerNorm's fp32 arithmetic, the GELU approximation: < 1e-6 relative.
   A difference before a bf16 store can move the stored value to its neighbour: one ulp = 2u.  Forward: u (P) + 2u (o
   re-rounded) + the later stores' flips -> 4u per row.  Backward adds P / dS (2u) and the re-rounding of dq / dk / dv
   (2u) -> 8u.  Held per query row (output), per context row (dctx / denc) and as a whole tensor; each weight gradient,
   and each column sum (mask token, every task embedding, norm and bias gradients) on its own as a whole tensor.
   Sensitivity: references with the neighbouring sample's ids, pos rows shifted by one patch, a dropped task embedding
   or a mask-token gradient summed over the visible rows must miss by >= 10x the budget.
3. The four *_ctx heads on four streams against the same calls serialised: fp32 reassociation only (1e-6 per row)."""
import ctypes
import os

import pytest
import torch

import pretrain_io_oracle as R
from multimae_b200 import _lib as L
from oracle import multimae_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -8                      # bf16 unit roundoff
FWD_ROW = 4 * U                    # decoder head output, per query row and whole tensor
GRAD_ROW = 8 * U                   # decoder head gradients, per row and whole tensor
SCATTER_TOL = 1e-6                 # class-embedding scatter, per row, of the sum of |terms|
STREAM_TOL = 1e-6                  # four streams against one


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(params=[0, 1], ids=["gelu_stream", "gelu_fused"])
def fuse_gelu(request):
    lib = L.lib()
    L.check(lib.mmae_set_fuse_gelu(request.param), "mmae_set_fuse_gelu")
    yield request.param
    lib.mmae_set_fuse_gelu(int(os.environ.get("MMAE_FUSE_GELU", "0")))      # the library's default


def _dy(shape, q, gen, dev, kmax=8):
    """dyadic values k / 2^q, |k| <= kmax, float64 on dev"""
    return (torch.randint(-kmax, kmax + 1, shape, generator=gen).double() / 2 ** q).to(dev)


def _exact(ref, absbound, q, what):
    """Premises of a bit-exact comparison: the reference is an fp32 value, and the sum of the magnitudes of the terms of
    every sum (a bound on each partial sum) is below 2^(23-q) for terms that are multiples of 2^-q."""
    assert torch.equal(ref, ref.float().double()), what + ": reference not representable in fp32"
    assert torch.equal(absbound * 2 ** q, torch.round(absbound * 2 ** q)), what + ": terms not multiples of 2^-q"
    assert float(absbound.max()) < 2.0 ** (23 - q), (what, float(absbound.max()), q)


def _masks(B, counts, T, kind, gen):
    """ids_keep / ids_restore from the oracle's sampler, shares Dirichlet(1) except:
      'dirichlet': sample 0 keeps only task 0's tokens, sample 1 only the last task's (Dirichlet-extreme draws);
      'head_extreme' (T > tokens per task): sample 0 keeps all of task 0's tokens, sample 1 none of them;
      'no_task1': task 1 keeps nothing anywhere."""
    n = len(counts)
    e = -torch.log(torch.rand(B, n, generator=gen))
    shares = e / e.sum(1, keepdim=True)
    if kind == "dirichlet":
        shares[0] = torch.eye(n)[0]
        if B > 1:
            shares[1] = torch.eye(n)[n - 1]
    elif kind == "head_extreme":
        x = counts[0] / T
        shares[0] = torch.tensor([x, 1 - x, 0.0])
        shares[1] = torch.tensor([0.0, 1 - x, x])
    else:
        shares[:] = torch.tensor([0.5, 0.0, 0.5])
    noises = [torch.rand(B, c, generator=gen) for c in counts]
    noise_all = torch.rand(B, sum(counts), generator=gen)
    _, keep, restore = O.sample_masks(shares, noises, noise_all, T)
    return keep, restore


def _report(name, errs):
    """print the worst fraction of budget of each check: errs = [(label, error, budget)]"""
    worst = max(errs, key=lambda e: e[1] / e[2])
    print("%s: worst %.3f of budget (%s: %.3g / %.3g)" % (name, worst[1] / worst[2], worst[0], worst[1], worst[2]))
    return worst[1] / worst[2]


# =============================================================================================================== embed
EMBED_CASES = {                    # S, B, T, G, D, mask kind
    "cfg2_b128": (224, 128, 98, 1, 768, "dirichlet"),
    "cfg5_b32": (448, 32, 392, 1, 768, "dirichlet"),
    "cfg4_d1024": (224, 8, 98, 1, 1024, "dirichlet"),
    "ragged_g1": (64, 3, 7, 1, 768, "dirichlet"),
    "ragged_g2": (64, 3, 7, 2, 768, "dirichlet"),
    "empty_task": (224, 16, 98, 1, 768, "no_task1"),
}


@pytest.mark.parametrize("case", list(EMBED_CASES))
def test_embed_bit_exact(dev, case):
    S, B, T, G, D, kind = EMBED_CASES[case]
    lib = L.lib()
    gen = torch.Generator().manual_seed(11)
    ncls, E = 133, 64
    n = (S // 16) ** 2
    # rgb (3 x 16^2 = 768), depth (256), semseg (64-wide class embedding, patch 4 on the S/4 label map: 1024)
    labels = torch.randint(0, 12, (B, S // 4, S // 4), generator=gen)       # mostly a few classes ...
    rare = torch.rand(labels.shape, generator=gen)
    labels[rare < 0.02] = torch.randint(12, ncls, (int((rare < 0.02).sum()),), generator=gen)   # ... some rare ones
    for bad, frac in ((-100, 0.01), (133, 0.005), (255, 0.01)):                     # ignore labels: embed as zeros
        labels[torch.rand(labels.shape, generator=gen) < frac] = bad
    tasks = [dict(image=_dy((B, 3, S, S), 3, gen, dev), patch=16),
             dict(image=_dy((B, 1, S, S), 3, gen, dev), patch=16),
             dict(labels=labels.to(dev), table=_dy((ncls, E), 3, gen, dev), patch=4)]
    K = [768, 256, E * 16]
    for t, tk in enumerate(tasks):
        tk["weight"] = _dy((D, K[t]), 4, gen, dev)
        tk["bias"] = _dy((D,), 4, gen, dev)
    pos = [_dy((n, D), 4, gen, dev) for _ in tasks]
    gtok = _dy((G, D), 4, gen, dev)
    keep, _ = _masks(B, [n] * 3, T, kind, gen)
    keep = keep.to(dev)

    lay = L.EmbedLayout()
    lay.num_tasks = 3
    for t in range(3):
        lay.grid_h[t] = lay.grid_w[t] = S // 16
        lay.tok_offset[t], lay.k_offset[t] = t * n, sum(K[:t])
        lay.patch[t] = tasks[t]["patch"]
        lay.channels[t] = (3, 1, E)[t]
        lay.is_semseg[t] = int(t == 2)
        lay.num_classes[t] = ncls if t == 2 else 0
    lay.tok_offset[3], lay.k_offset[3] = 3 * n, sum(K)
    f32 = lambda x: x.float().contiguous()
    data = [f32(tasks[0]["image"]), f32(tasks[1]["image"]), tasks[2]["labels"].contiguous()]
    w32 = [f32(tk["weight"]) for tk in tasks]
    b32 = [f32(tk["bias"]) for tk in tasks]
    p32 = [f32(p) for p in pos]
    table32, g32 = f32(tasks[2]["table"]), f32(gtok)
    ins, prm, grd = L.EmbedInputs(), L.EmbedParams(), L.EmbedGrads()
    for t in range(3):
        ins.data[t] = data[t].data_ptr()
        prm.weight[t], prm.bias[t], prm.pos[t] = w32[t].data_ptr(), b32[t].data_ptr(), p32[t].data_ptr()
    ins.class_emb[2] = table32.data_ptr()
    prm.global_tokens = g32.data_ptr()
    saved = torch.empty(lib.mmae_embed_saved_bytes(ctypes.byref(lay), B, T, D), dtype=torch.uint8, device=dev)
    ws = torch.empty(lib.mmae_embed_workspace_bytes(ctypes.byref(lay), B, T, D), dtype=torch.uint8, device=dev)
    x = torch.empty(B, T + G, D, device=dev)
    L.check(lib.mmae_embed_forward(ctypes.byref(lay), ctypes.byref(ins), ctypes.byref(prm), keep.data_ptr(), B, T, G, D,
                                   x.data_ptr(), saved.data_ptr(), ws.data_ptr(), L.current_stream()), "embed forward")
    # gradients accumulate onto non-zero values
    prior = {"w": [_dy((D, k), 4, gen, dev) for k in K], "b": [_dy((D,), 4, gen, dev) for _ in K],
             "cls": _dy((ncls, E), 4, gen, dev), "g": _dy((G, D), 4, gen, dev)}
    gw, gb = [f32(v) for v in prior["w"]], [f32(v) for v in prior["b"]]
    gcls, gg = f32(prior["cls"]), f32(prior["g"])
    for t in range(3):
        grd.weight[t], grd.bias[t] = gw[t].data_ptr(), gb[t].data_ptr()
    grd.class_emb[2], grd.global_tokens = gcls.data_ptr(), gg.data_ptr()
    dx = _dy((B, T + G, D), 4, gen, dev)
    dx32 = f32(dx)
    L.check(lib.mmae_embed_backward(ctypes.byref(lay), ctypes.byref(ins), ctypes.byref(prm), ctypes.byref(grd),
                                    keep.data_ptr(), B, T, G, D, dx32.data_ptr(), saved.data_ptr(), ws.data_ptr(),
                                    L.current_stream()), "embed backward")
    torch.cuda.synchronize()

    ref = R.embed_forward(tasks, pos, gtok, keep)
    abs_tasks = [dict(tk, image=tk["image"].abs(), weight=tk["weight"].abs(), bias=tk["bias"].abs()) if "image" in tk else
                 dict(tk, table=tk["table"].abs(), weight=tk["weight"].abs(), bias=tk["bias"].abs()) for tk in tasks]
    _exact(ref, R.embed_forward(abs_tasks, [p.abs() for p in pos], gtok.abs(), keep), 7, "embed forward")
    assert torch.equal(x.double(), ref), (case, float((x.double() - ref).abs().max()))

    grads, dg = R.embed_backward(tasks, pos, keep, dx, G)
    agrads, adg = R.embed_backward(abs_tasks, pos, keep, dx.abs(), G)
    for t in range(3):
        rw, rbias = prior["w"][t] + grads[t]["weight"], prior["b"][t] + grads[t]["bias"]
        _exact(rw, prior["w"][t].abs() + agrads[t]["weight"], 7, "dW_%d" % t)
        _exact(rbias, prior["b"][t].abs() + agrads[t]["bias"], 4, "db_%d" % t)
        assert torch.equal(gw[t].double(), rw), (case, t, "weight", float((gw[t].double() - rw).abs().max()))
        assert torch.equal(gb[t].double(), rbias), (case, t, "bias", float((gb[t].double() - rbias).abs().max()))
    _exact(prior["g"] + dg, prior["g"].abs() + adg, 4, "dglobal")
    assert torch.equal(gg.double(), prior["g"] + dg), case
    if kind == "no_task1":                                     # a task without kept tokens: its gradients stay as they were
        assert bool((keep < n).any()) and not bool(((keep >= n) & (keep < 2 * n)).any())
        assert torch.equal(gw[1].double(), prior["w"][1]) and torch.equal(gb[1].double(), prior["b"][1])
    # dA = bf16(dC W_t): its fp32 sum is exact, the scatter of mixed exponents is not
    dt = torch.zeros(B, 3 * n, D, dtype=torch.float64, device=dev)
    dt.scatter_(1, keep[..., None].expand(B, T, D), dx.abs()[:, :T])
    _exact(dt[:, 2 * n:] @ tasks[2]["weight"].abs(), dt[:, 2 * n:] @ tasks[2]["weight"].abs(), 8, "dA")
    rc, scale = prior["cls"] + grads[2]["class_emb"], grads[2]["class_emb_abs"]
    err = (gcls.double() - rc).norm(dim=1)
    bound = SCATTER_TOL * scale.norm(dim=1)
    untouched = scale.norm(dim=1) == 0
    assert torch.equal(gcls.double()[untouched], prior["cls"][untouched]), case
    _report("embed %s class_emb" % case, [("row %d" % i, float(err[i]), float(bound[i])) for i in range(ncls)
                                          if not untouched[i]])
    assert bool((err <= bound).all()), (case, int((err > bound).sum()), float((err / bound.clamp_min(1e-30)).max()))


# ============================================================================================================= ctxproj
@pytest.mark.parametrize("layout", ["in_place_mirror", "gathered"])
def test_ctxproj_bit_exact(dev, layout):
    lib = L.lib()
    gen = torch.Generator().manual_seed(12)
    B, T, De, dims = 128, 98, 768, [256, 256, 256, 256]
    rows, Dsum = B * (T + 1), sum(dims)
    enc = _dy((rows, De), 3, gen, dev)
    W = [_dy((d, De), 4, gen, dev) for d in dims]
    bias = [_dy((d,), 4, gen, dev) for d in dims]
    dctx = _dy((rows, Dsum), 4, gen, dev)
    prior = [_dy((d, De), 4, gen, dev) for d in dims]
    mirror = None
    if layout == "in_place_mirror":                # adjacent parameters, gradient slots and a registered bf16 twin
        wflat = torch.cat(W).float().contiguous()
        bflat = torch.cat(bias).float().contiguous()
        gflat = torch.cat(prior).float().contiguous()
        w32, b32, g32 = list(wflat.split(dims)), list(bflat.split(dims)), list(gflat.split(dims))
        mirror = wflat.to(torch.bfloat16).contiguous()
        L.check(lib.mmae_weight_mirror_register(wflat.data_ptr(), mirror.data_ptr(), wflat.numel()), "mirror")
    else:                                          # separate tensors, no twin: gathered and cast per call
        w32 = [w.float().contiguous() for w in W]
        b32 = [b.float().contiguous() for b in bias]
        g32 = [g.float().contiguous() for g in prior]
    try:
        prm, grd = L.CtxProjParams(), L.CtxProjGrads()
        prm.num = len(dims)
        for i, d in enumerate(dims):
            prm.dim[i], prm.weight[i], prm.bias[i], grd.weight[i] = d, w32[i].data_ptr(), b32[i].data_ptr(), g32[i].data_ptr()
        enc32 = enc.float().contiguous()
        saved = torch.empty(lib.mmae_ctxproj_saved_bytes(rows, De, Dsum), dtype=torch.uint8, device=dev)
        ctx = torch.empty(rows, Dsum, device=dev)
        L.check(lib.mmae_ctxproj_forward(enc32.data_ptr(), rows, De, ctypes.byref(prm), ctx.data_ptr(), saved.data_ptr(),
                                         L.current_stream()), "ctxproj forward")
        db16 = dctx.to(torch.bfloat16).contiguous()
        denc = torch.full((rows, De), 7.0, device=dev)                 # written, not accumulated
        L.check(lib.mmae_ctxproj_backward(rows, De, ctypes.byref(prm), ctypes.byref(grd), db16.data_ptr(), denc.data_ptr(),
                                          saved.data_ptr(), L.current_stream()), "ctxproj backward")
        torch.cuda.synchronize()
    finally:
        if mirror is not None:
            lib.mmae_weight_mirror_register(wflat.data_ptr(), None, 0)
    ref = R.ctxproj_forward(enc, W, bias)
    _exact(ref, R.ctxproj_forward(enc.abs(), [w.abs() for w in W], [b.abs() for b in bias]), 7, "ctx")
    assert torch.equal(ctx.double(), ref), layout
    dW, denc_ref = R.ctxproj_backward(enc, W, dctx)
    adW, adenc = R.ctxproj_backward(enc.abs(), [w.abs() for w in W], dctx.abs())
    _exact(denc_ref, adenc, 8, "denc")
    assert torch.equal(denc.double(), denc_ref), layout
    for i in range(len(dims)):
        _exact(prior[i] + dW[i], prior[i].abs() + adW[i], 7, "dW")
        assert torch.equal(g32[i].double(), prior[i] + dW[i]), (layout, i)


# ============================================================================================================= dectail
@pytest.mark.parametrize("S,B", [(224, 128), (448, 32)])
@pytest.mark.parametrize("C,P", [(3, 16), (1, 16), (133, 4)])
def test_dectail_bit_exact(dev, S, B, C, P):
    lib = L.lib()
    gen = torch.Generator().manual_seed(13)
    Dd = 256
    nh = nw = S // 16
    x = _dy((B, nh * nw, Dd), 3, gen, dev)
    w = _dy((C * P * P, Dd), 4, gen, dev)
    b = _dy((C * P * P,), 4, gen, dev)
    dpred = _dy((B, C, nh * P, nw * P), 4, gen, dev)
    prior_w, prior_b = _dy(w.shape, 4, gen, dev), _dy(b.shape, 4, gen, dev)
    x32, w32, b32, dp32 = (t.float().contiguous() for t in (x, w, b, dpred))
    gw, gb = prior_w.float().contiguous(), prior_b.float().contiguous()
    dims = (B, nh, nw, Dd, C, P)
    saved = torch.empty(lib.mmae_dectail_saved_bytes(*dims), dtype=torch.uint8, device=dev)
    ws = torch.empty(lib.mmae_dectail_workspace_bytes(*dims), dtype=torch.uint8, device=dev)
    pred = torch.empty(B, C, nh * P, nw * P, device=dev)
    dx = torch.empty(B, nh * nw, Dd, device=dev)
    st = L.current_stream()
    L.check(lib.mmae_dectail_forward(x32.data_ptr(), *dims, w32.data_ptr(), b32.data_ptr(), pred.data_ptr(),
                                     saved.data_ptr(), ws.data_ptr(), st), "dectail forward")
    L.check(lib.mmae_dectail_backward(dp32.data_ptr(), *dims, w32.data_ptr(), gw.data_ptr(), gb.data_ptr(), dx.data_ptr(),
                                      saved.data_ptr(), ws.data_ptr(), st), "dectail backward")
    torch.cuda.synchronize()
    _exact(x.abs() @ w.abs().t() + b.abs(), x.abs() @ w.abs().t() + b.abs(), 7, "out_proj")
    ref = R.dectail_forward(x, w, b, C, nh, nw, P)
    assert torch.equal(pred.double(), ref), float((pred.double() - ref).abs().max())
    dW, db, dxr = R.dectail_backward(x, w, dpred, P)
    adW, adb, adx = R.dectail_backward(x.abs(), w.abs(), dpred.abs(), P)
    _exact(prior_w + dW, prior_w.abs() + adW, 7, "dW")
    _exact(prior_b + db, prior_b.abs() + adb, 4, "db")
    _exact(dxr, adx, 8, "dx")
    assert torch.equal(gw.double(), prior_w + dW)
    assert torch.equal(gb.double(), prior_b + db)
    assert torch.equal(dx.double(), dxr)


# ======================================================================================================== decoder head
HEAD_W = ["q_w", "kv_w", "proj_w", "fc1_w", "fc2_w"]
HEAD_VEC = ["context_norm_w", "context_norm_b", "query_norm_w", "query_norm_b", "out_norm_w", "out_norm_b", "q_b", "kv_b",
            "proj_b", "fc1_b", "fc2_b"]
DD, HEADS, HIDDEN, DE, EPS = 256, 8, 1024, 768, 1e-6


def _head_inputs(B, n, T, mode, own, gen, dev, ctx_mode):
    """Parameters and inputs of one decoder head (float64 on dev); the q / k weights are scaled up so that attention is
    peaked and the output depends on which query row is which."""
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64).to(dev)
    prm = {"mask_token": r(DD), "pos": r(n, DD), "task_emb": [r(DD) for _ in range(4)]}
    for nm in ("context_norm", "query_norm", "out_norm"):
        prm[nm + "_w"], prm[nm + "_b"] = 1 + 0.1 * r(DD), 0.1 * r(DD)
    prm["q_w"] = r(DD, DD) * 1.5 / DD ** 0.5
    prm["kv_w"] = torch.cat([r(DD, DD) * 1.5, r(DD, DD)]) / DD ** 0.5
    prm["proj_w"], prm["fc1_w"], prm["fc2_w"] = r(DD, DD) / DD ** 0.5, r(HIDDEN, DD) / DD ** 0.5, r(DD, HIDDEN) / HIDDEN ** 0.5
    for nm, d in (("q_b", DD), ("kv_b", 2 * DD), ("proj_b", DD), ("fc1_b", HIDDEN), ("fc2_b", DD)):
        prm[nm] = 0.1 * r(d)
    if not ctx_mode:
        prm["proj_context_w"], prm["proj_context_b"] = r(DD, DE) / DE ** 0.5, 0.1 * r(DD)
    # round every parameter to fp32 once: the kernels read the fp32 values
    prm = {k: ([t.float().double() for t in v] if isinstance(v, list) else v.float().double()) for k, v in prm.items()}
    keep, restore = _masks(B, [n] * 3, T, "head_extreme" if T > n else "dirichlet", gen)
    ix = {"num_visible": T, "num_queries": n, "tok_offset": [0, n, 2 * n, 3 * n], "own_task": own, "query_mode": mode,
          "ids_keep": keep.to(dev), "ids_restore": restore.to(dev)}
    return prm, ix


def _head_struct(ix, B):
    s = L.DecoderIndex()
    s.batch, s.dim, s.num_visible, s.num_global = B, DD, ix["num_visible"], 1
    s.num_queries, s.total_tokens, s.num_tasks = ix["num_queries"], ix["tok_offset"][-1], 3
    s.own_task, s.query_mode = ix["own_task"], ix["query_mode"]
    for i, o in enumerate(ix["tok_offset"]):
        s.tok_offset[i] = o
    s.ids_keep, s.ids_restore = ix["ids_keep"].data_ptr(), ix["ids_restore"].data_ptr()
    return s


class _Head:
    """fp32 device copies of one head's parameters, gradient slots and buffers, and the ctypes structs over them."""

    def __init__(self, prm, ix, B, De, dev):
        self.p32 = {k: ([t.float().contiguous() for t in v] if isinstance(v, list) else v.float().contiguous())
                    for k, v in prm.items()}
        self.g32 = {k: torch.zeros_like(v) for k, v in self.p32.items() if k not in ("pos", "task_emb")}
        self.g32["task_emb"] = [torch.zeros_like(t) for t in self.p32["task_emb"]]
        self.g32.setdefault("proj_context_b", torch.zeros(DD, device=dev))     # *_ctx heads: the bias gradient only
        self.ix = _head_struct(ix, B)
        self.prm, self.grd = L.DecHeadParams(), L.DecHeadGrads()
        for k, v in self.p32.items():
            if k == "task_emb":
                for t in range(4):
                    self.prm.task_emb[t] = v[t].data_ptr()
                    self.grd.task_emb[t] = self.g32["task_emb"][t].data_ptr()
            else:
                setattr(self.prm, k, v.data_ptr())
        for k, v in self.g32.items():
            if k != "task_emb":
                setattr(self.grd, k, v.data_ptr())
        lib = L.lib()
        self.saved = torch.empty(lib.mmae_dechead_saved_bytes(ctypes.byref(self.ix), De, HEADS, HIDDEN), dtype=torch.uint8,
                                 device=dev)
        self.ws = torch.empty(lib.mmae_dechead_workspace_bytes(ctypes.byref(self.ix), De, HEADS, HIDDEN), dtype=torch.uint8,
                              device=dev)
        self.out = torch.empty(B, ix["num_queries"], DD, device=dev)

    def forward_ctx(self, ctx_all, offset, st):
        L.check(L.lib().mmae_dechead_forward_ctx(ctx_all.data_ptr() + 4 * offset, ctx_all.shape[1], ctypes.byref(self.ix),
                                                 HEADS, HIDDEN, EPS, ctypes.byref(self.prm), self.out.data_ptr(),
                                                 self.saved.data_ptr(), self.ws.data_ptr(), st), "dechead forward_ctx")

    def backward_ctx(self, dout, dctx_all, offset, st):
        L.check(L.lib().mmae_dechead_backward_ctx(ctypes.byref(self.ix), HEADS, HIDDEN, ctypes.byref(self.prm),
                                                  ctypes.byref(self.grd), dout.data_ptr(), dctx_all.data_ptr() + 2 * offset,
                                                  dctx_all.shape[1], self.saved.data_ptr(), self.ws.data_ptr(), st),
                "dechead backward_ctx")


def _rel_rows(got, ref):
    """(whole-tensor relative L2, worst per-row relative L2) over the last dimension"""
    got, ref = got.double(), ref.double()
    got, ref = (got.flatten(0, -2), ref.flatten(0, -2)) if ref.dim() > 1 else (got[None], ref[None])
    d = got - ref
    rows = d.norm(dim=1) / ref.norm(dim=1).clamp_min(1e-300)
    return float(d.norm() / ref.norm()), float(rows.max())


PER_ROW = ("x_out", "dctx", "denc")   # per query row, per context row


def _head_checks(got, ref):
    """[(label, error, budget)] for every output / gradient tensor as a whole, and per row for the activation-shaped ones.
    A row of a weight gradient is a sum over every query (or context) row of products of varying sign: its norm can lie
    far below the magnitude of its terms, which is what the per-element bound scales with, so it is held as a whole."""
    out = []
    for k, (g, r) in got.items():
        whole, row = _rel_rows(g, r)
        budget = FWD_ROW if k == "x_out" else GRAD_ROW
        out.append((k, whole, budget))
        if k in PER_ROW:
            out.append((k + " row", row, budget))
    return out


HEAD_CASES = {            # B, tokens per task, visible, query mode, own task, ctx offset (None: the encoder-output entry)
    "mode0_own0_B1": (1, 196, 98, 0, 0, 0),
    "mode0_own0_extreme": (3, 16, 20, 0, 0, 0),
    "mode0_own1_off256": (3, 16, 20, 0, 1, 256),
    "mode0_own2_enc": (3, 16, 20, 0, 2, None),
    "mode1_noq_off768": (3, 16, 20, 1, -1, 768),
    "mode1_spare_enc": (3, 16, 20, 1, 3, None),
    "448_B4": (4, 784, 392, 0, 0, 256),
    "cfg2_B128": (128, 196, 98, 0, 0, 0),
}


def _run_head_case(dev, case, fuse, mutations=()):
    B, n, T, mode, own, off = HEAD_CASES[case]
    gen = torch.Generator().manual_seed(21)
    ctx_mode = off is not None
    prm, ix = _head_inputs(B, n, T, mode, own, gen, dev, ctx_mode)
    Nc = T + 1
    dout = torch.randn(B, n, DD, generator=gen, dtype=torch.float64).float().double().to(dev)
    De = 0 if ctx_mode else DE
    h = _Head(prm, ix, B, De, dev)
    lib, st = L.lib(), L.current_stream()
    dout32 = dout.float().contiguous()
    if ctx_mode:
        ctx_all = torch.randn(B * Nc, 1024, generator=gen).to(dev)
        dctx_all = torch.zeros(B * Nc, 1024, dtype=torch.bfloat16, device=dev)
        h.forward_ctx(ctx_all, off, st)
        h.backward_ctx(dout32, dctx_all, off, st)
        src = ctx_all[:, off:off + DD].double().reshape(B, Nc, DD)
    else:
        enc = torch.randn(B, Nc, DE, generator=gen).to(dev)
        denc = torch.randn(B, Nc, DE, generator=gen).to(dev)                 # accumulated onto
        denc0 = denc.double()
        L.check(lib.mmae_dechead_forward(enc.data_ptr(), DE, ctypes.byref(h.ix), HEADS, HIDDEN, EPS, ctypes.byref(h.prm),
                                         h.out.data_ptr(), h.saved.data_ptr(), h.ws.data_ptr(), st), "dechead forward")
        L.check(lib.mmae_dechead_backward(enc.data_ptr(), DE, ctypes.byref(h.ix), HEADS, HIDDEN, ctypes.byref(h.prm),
                                          ctypes.byref(h.grd), dout32.data_ptr(), denc.data_ptr(), h.saved.data_ptr(),
                                          h.ws.data_ptr(), st), "dechead backward")
        src = enc.double()
    torch.cuda.synchronize()

    def reference(mutate=None):
        leaves = {k: ([t.clone().requires_grad_(True) for t in v] if k == "task_emb" else
                      v.clone().requires_grad_(k != "pos")) for k, v in prm.items()}
        s = src.clone().requires_grad_(True)
        c = s if ctx_mode else R.rb(R.rf(s) @ R.rf(leaves["proj_context_w"]).t()) + leaves["proj_context_b"]
        x_out, queries = R.dechead_reference(c, ix, leaves, HEADS, EPS, fuse, dout, mutate)
        ref = {"x_out": x_out}
        for k in HEAD_W + HEAD_VEC + ["mask_token"] + ([] if ctx_mode else ["proj_context_w", "proj_context_b"]):
            ref[k] = leaves[k].grad
        used = set(range(3)) | ({own} if own >= 0 else set())
        for t in used:
            ref["task_emb.%d" % t] = leaves["task_emb"][t].grad
        if ctx_mode:
            ref["dctx"] = R.bf16(s.grad).reshape(B * Nc, DD)
            ref["proj_context_b"] = s.grad.sum((0, 1))
        else:
            ref["denc"] = denc0 + s.grad
        return ref, queries

    ref, queries = reference()
    got = {"x_out": h.out}
    for k in ref:
        if k.startswith("task_emb."):
            got[k] = h.g32["task_emb"][int(k.split(".")[1])]
        elif k == "dctx":
            got[k] = dctx_all[:, off:off + DD]
        elif k == "denc":
            got[k] = denc
        elif k != "x_out":
            got[k] = h.g32[k]
    if ctx_mode:                                             # the other adapters' segments are not written
        rest = torch.cat([dctx_all[:, :off], dctx_all[:, off + DD:]], 1)
        assert not bool(rest.any())
    if own >= 0 and own < 3:
        assert not bool(h.g32["task_emb"][3].any())        # the spare slot gets nothing unless it is the query task
    pairs = {k: (got[k], ref[k]) for k in ref}
    errs = _head_checks(pairs, ref)
    frac = _report("dechead %s fuse=%d" % (case, fuse), errs)
    assert frac <= 1.0, [e for e in errs if e[1] > e[2]]

    for m in mutations:                                     # plausibly wrong references must fail by >= 10x
        if m == "mask_from_visible":
            rank = ix["ids_restore"][:, ix["tok_offset"][own]:ix["tok_offset"][own] + n]
            wrong = dict(ref, mask_token=queries.grad[rank < T].sum(0))
        else:
            wrong, _ = reference(m)
        wf = max(e[1] / e[2] for e in _head_checks({k: (got[k], wrong[k]) for k in wrong}, wrong))
        print("  wrong reference %s: %.1f x budget" % (m, wf))
        assert wf >= 10.0, (m, wf)


@pytest.mark.parametrize("case", [c for c in HEAD_CASES if c != "cfg2_B128"])
def test_dechead_against_rounding_reference(dev, fuse_gelu, case):
    muts = ()
    if case == "mode0_own0_extreme":
        muts = ("neighbour_ids", "pos_shift", "drop_task_emb", "mask_from_visible")
    _run_head_case(dev, case, fuse_gelu, muts)


def test_dechead_bench_batch(dev, fuse_gelu):
    _run_head_case(dev, "cfg2_B128", fuse_gelu)


def test_dechead_extreme_masks_present(dev):
    """The small cases' draws include a sample whose own task is fully visible and one where it is fully masked."""
    B, n, T, mode, own, _ = HEAD_CASES["mode0_own0_extreme"]
    _, ix = _head_inputs(B, n, T, mode, own, torch.Generator().manual_seed(21), dev, True)
    vis = (ix["ids_restore"][:, :n] < T).sum(1)
    assert int(vis[0]) == 16 and int(vis[1]) == 0, vis


# ===================================================================================================== four streams
def test_four_ctx_heads_on_four_streams(dev):
    """The four *_ctx heads forward and backward each on its own stream, joined by events, against the same calls on one
    stream: every output and gradient within fp32 reassociation (per row)."""
    B, n, T = 16, 196, 98
    gen = torch.Generator().manual_seed(31)
    heads = []
    for i in range(4):                 # one mask draw for all four, as in a step; own task 0, 1, 2 and a mask-token head
        prm, ix = _head_inputs(B, n, T, 0, 0, gen, dev, True)
        ix0 = heads[0][1] if heads else ix
        heads.append((prm, dict(ix0, own_task=i if i < 3 else -1, query_mode=0 if i < 3 else 1)))
    ctx_all = torch.randn(B * (T + 1), 1024, generator=gen).to(dev)
    douts = [torch.randn(B, n, DD, generator=gen).to(dev) for _ in range(4)]

    def run(streams):
        hs = [_Head(p, ix, B, 0, dev) for p, ix in heads]
        dctx = torch.zeros(B * (T + 1), 1024, dtype=torch.bfloat16, device=dev)
        main = torch.cuda.current_stream()
        ready = main.record_event()
        for i, h in enumerate(hs):
            s = streams[i] if streams else main
            s.wait_event(ready)
            with torch.cuda.stream(s):
                h.forward_ctx(ctx_all, 256 * i, s.cuda_stream)
        for s in streams or ():
            main.wait_stream(s)
        ready = main.record_event()
        for i, h in enumerate(hs):
            s = streams[i] if streams else main
            s.wait_event(ready)
            with torch.cuda.stream(s):
                h.backward_ctx(douts[i], dctx, 256 * i, s.cuda_stream)
        for s in streams or ():
            main.wait_stream(s)
        torch.cuda.synchronize()
        return hs, dctx

    one, dctx1 = run(None)
    four, dctx4 = run([torch.cuda.Stream(device=dev) for _ in range(4)])
    errs = [("dctx", _rel_rows(dctx4.float(), dctx1.double())[1], STREAM_TOL)]
    for i, (a, b) in enumerate(zip(one, four)):
        errs.append(("x_out %d" % i, _rel_rows(b.out, a.out.double())[1], STREAM_TOL))
        for k, v in a.g32.items():
            for j, (ga, gb) in enumerate(zip(v, b.g32[k]) if k == "task_emb" else [(v, b.g32[k])]):
                if bool(ga.any()):
                    errs.append(("%s %d.%d" % (k, i, j), _rel_rows(gb, ga.double())[1], STREAM_TOL))
                else:
                    assert not bool(gb.any()), (k, i, j)
    frac = _report("four streams", errs)
    assert frac <= 1.0, [e for e in errs if e[1] > e[2]]

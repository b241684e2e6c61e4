"""Float64 references of the pre-training input / output side (tests/test_cuda_pretrain_io.py).

* embed / ctxproj / dectail: plain float64 of the module's arithmetic.  The tests feed dyadic values chosen so that every
  fp32 sum the kernels form is exact; bf16 roundings of exact values are applied where the kernels store bf16.
* decoder head: float64 with a bf16 rounding wherever dechead_forward_impl / dechead_backward_impl store a bf16 tensor
  (RoundFwd on values, RoundBwd on the gradient operands), in both GELU modes of mmae_set_fuse_gelu; with round=False,
  plain float64 (the fp32 tier, mmae_dechead_f32_*).

Everything runs on whatever device its inputs are on (the bench-sized cases run it on the GPU in float64)."""
import math

import torch
import torch.nn.functional as F


def bf16(x):
    """Round-to-nearest-even to bf16, returned in x's dtype."""
    return x.to(torch.bfloat16).to(x.dtype)


def patchify(img, P):
    """[B, C, nh*P, nw*P] -> [B, nh*nw, C*P*P] in conv-weight (c, py, px) order."""
    B, C, H, W = img.shape
    nh, nw = H // P, W // P
    return img.reshape(B, C, nh, P, nw, P).permute(0, 2, 4, 1, 3, 5).reshape(B, nh * nw, C * P * P)


def unpatchify(tok, C, nh, nw, P):
    """[B, nh*nw, C*P*P] -> [B, C, nh*P, nw*P]."""
    B = tok.shape[0]
    return tok.reshape(B, nh, nw, C, P, P).permute(0, 3, 1, 4, 2, 5).reshape(B, C, nh * P, nw * P)


def semseg_image(labels, table):
    """nn.Embedding lookup of a label map [B, H, W] -> [B, E, H, W]; labels outside [0, num_classes) embed as zeros."""
    K = table.shape[0]
    ok = (labels >= 0) & (labels < K)
    emb = table[labels.clamp(0, K - 1)] * ok[..., None].to(table.dtype)
    return emb.permute(0, 3, 1, 2)


# --------------------------------------------------------------------------------------------------------------- embed
def embed_tokens(tasks, pos):
    """tasks: list of dicts (image [B,C,H,W] float64 or labels [B,H,W] int64 + table, weight [D,K], bias [D], patch).
    Returns (tokens [B, N_total, D], patches per task [B, N_t, K_t])."""
    toks, patches = [], []
    for t, tk in enumerate(tasks):
        img = semseg_image(tk["labels"], tk["table"]) if "labels" in tk else tk["image"]
        a = patchify(img, tk["patch"])
        patches.append(a)
        toks.append(a @ tk["weight"].t() + tk["bias"] + pos[t])
    return torch.cat(toks, 1), patches


def embed_forward(tasks, pos, global_tokens, ids_keep):
    tok, _ = embed_tokens(tasks, pos)
    B, T = ids_keep.shape
    kept = torch.gather(tok, 1, ids_keep[..., None].expand(B, T, tok.shape[2]))
    return torch.cat([kept, global_tokens.expand(B, -1, -1)], 1)


def embed_backward(tasks, pos, ids_keep, dx, G):
    """Gradients of embed_forward for dx [B, T+G, D]: per task dW, db, and for semseg tasks the class-embedding gradient
    (dA = dC W_t rounded to bf16 as the kernel stores it, then scattered by label) together with the same scatter of |dA|
    (the magnitude scale of each table entry's fp32 sum); plus the global-token gradient."""
    B, T = ids_keep.shape
    D = dx.shape[2]
    counts = [patchify(semseg_image(tk["labels"], tk["table"]) if "labels" in tk else tk["image"], tk["patch"]).shape[1]
              for tk in tasks]
    dtok = torch.zeros(B, sum(counts), D, dtype=dx.dtype, device=dx.device)
    dtok.scatter_(1, ids_keep[..., None].expand(B, T, D), dx[:, :T])
    _, patches = embed_tokens(tasks, pos)
    out, off = [], 0
    for t, tk in enumerate(tasks):
        dt = dtok[:, off:off + counts[t]]
        off += counts[t]
        g = {"weight": torch.einsum("bnd,bnk->dk", dt, patches[t]), "bias": dt.sum((0, 1))}
        if "labels" in tk:
            P, labels, table = tk["patch"], tk["labels"], tk["table"]
            E = table.shape[1]
            nh, nw = labels.shape[1] // P, labels.shape[2] // P
            dA = bf16(dt @ tk["weight"])
            g["class_emb"] = _scatter_classes(unpatchify(dA, E, nh, nw, P), labels, table.shape[0])
            g["class_emb_abs"] = _scatter_classes(unpatchify(dA.abs(), E, nh, nw, P), labels, table.shape[0])
        out.append(g)
    return out, dx[:, T:].sum(0)


def _scatter_classes(img, labels, K):
    """sum over pixels with label k in [0, K) of img[b, :, y, x] -> [K, E]"""
    E = img.shape[1]
    ok = (labels >= 0) & (labels < K)
    vals = img.permute(0, 2, 3, 1)[ok]
    out = torch.zeros(K, E, dtype=img.dtype, device=img.device)
    return out.index_add_(0, labels[ok], vals)


# ----------------------------------------------------------------------------------------------------- ctxproj / tail
def ctxproj_forward(enc, weights, biases):
    return bf16(enc) @ torch.cat(weights).t() + torch.cat(biases)


def ctxproj_backward(enc, weights, dctx):
    """(per-adapter dW, denc) for the bf16 context gradient dctx [rows, sum Dd]."""
    dW = dctx.t() @ bf16(enc)
    return list(torch.split(dW, [w.shape[0] for w in weights])), dctx @ torch.cat(weights)


def dectail_forward(x, weight, bias, C, nh, nw, P):
    """out_proj in half precision (bf16 output), then un-patchify."""
    return unpatchify(bf16(x @ weight.t() + bias), C, nh, nw, P)


def dectail_backward(x, weight, dpred, P):
    dy = patchify(dpred, P)
    return dy.flatten(0, 1).t() @ x.flatten(0, 1), dy.sum((0, 1)), dy @ weight


# ------------------------------------------------------------------------------------------------------ decoder head
class RoundFwd(torch.autograd.Function):
    """bf16 rounding of a stored value; the gradient passes through unchanged."""

    @staticmethod
    def forward(ctx, x):
        return bf16(x)

    @staticmethod
    def backward(ctx, g):
        return g


class RoundBwd(torch.autograd.Function):
    """Identity on the value; the gradient is rounded to bf16 (a bf16 gradient operand of the kernels)."""

    @staticmethod
    def forward(ctx, x):
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        return bf16(g)


rf, rb = RoundFwd.apply, RoundBwd.apply


def roundings(round):
    """(rf, rb), or two identities for the plain float64 reference (round=False)"""
    return (rf, rb) if round else ((lambda x: x), (lambda x: x))


class Attention(torch.autograd.Function):
    """softmax(q k^T s) v per head, float64, with the backward's row term delta = rowsum(dO * O) formed from the stored
    bf16 output O as the kernel forms it (not from the float64 P)."""

    @staticmethod
    def forward(ctx, q, k, v, scale):
        p = torch.softmax(q @ k.transpose(-1, -2) * scale, -1)
        o = p @ v
        ctx.save_for_backward(q, k, v, p, bf16(o))
        ctx.scale = scale
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, p, o_b = ctx.saved_tensors
        dv = p.transpose(-1, -2) @ do
        dp = do @ v.transpose(-1, -2)
        ds = p * (dp - (do * o_b).sum(-1, keepdim=True))
        return ds @ k * ctx.scale, ds.transpose(-1, -2) @ q * ctx.scale, dv, None


def attention(q, k, v, scale, round=True):
    """Attention with the kernels' backward row term (round=True), else plain float64 autograd."""
    if round:
        return Attention.apply(q, k, v, scale)
    return torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _ln(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def build_queries_context(ctx, ix, mask_token, task_emb, pos, mutate=None):
    """dec_build_kernel: ctx [B, T+G, Dd] -> (queries [B, P, Dd], context [B, T+G, Dd]).  `mutate` names a deliberately
    wrong variant (the tests' sensitivity checks)."""
    B, Nc, Dd = ctx.shape
    T, P = ix["num_visible"], ix["num_queries"]
    tok_off, own, mode = ix["tok_offset"], ix["own_task"], ix["query_mode"]
    ids_keep, ids_restore = ix["ids_keep"], ix["ids_restore"]
    ntask = len(tok_off) - 1
    dev = ctx.device
    pos_q = pos[:P]
    if mutate == "pos_shift":
        pos_q = torch.roll(pos, 1, 0)[:P]
    if mode == 0:
        restore = ids_restore
        if mutate == "neighbour_ids":
            restore = torch.roll(ids_restore, 1, 0)
        rank = restore[:, tok_off[own]:tok_off[own] + P]                     # [B, P]
        vis = rank < T
        src = torch.gather(ctx, 1, rank.clamp(max=T - 1)[..., None].expand(B, P, Dd))
        base = torch.where(vis[..., None], src, mask_token.reshape(1, 1, Dd).expand(B, P, Dd))
    else:
        base = mask_token.reshape(1, 1, Dd).expand(B, P, Dd)
    q = base + pos_q
    if own >= 0 and mutate != "drop_task_emb":
        q = q + task_emb[own].reshape(1, 1, Dd)
    # context: visible tokens get their task's embedding and their patch's position row; global tokens pass through
    g = ids_keep                                                              # [B, T]
    task = torch.zeros_like(g)
    for t in range(1, ntask):
        task = torch.where(g >= tok_off[t], torch.full_like(g, t), task)
    offs = torch.tensor(tok_off[:ntask], device=dev)[task]
    te = torch.stack([task_emb[t].reshape(Dd) for t in range(ntask)])[task]   # [B, T, Dd]
    c_vis = ctx[:, :T] + pos[g - offs] + te
    context = torch.cat([c_vis, ctx[:, T:]], 1)
    return q, context


def dechead_reference(ctx, ix, prm, H, eps, fuse_gelu, dout, mutate=None, round=True):
    """Forward and backward of the decoder head from the fp32 context projection `ctx` [B, T+G, Dd] (a float64 leaf, or
    the caller's rounded proj_context of an encoder-output leaf).  prm: float64 leaves (requires_grad) named as
    DecHeadParams' fields, task_emb a list.  Runs backward(dout); returns (x_out, queries) - queries with its .grad.
    round=False: no bf16 rounding anywhere and plain attention (fuse_gelu then has no effect)."""
    rf, rb = roundings(round)
    B, Nc, Dd = ctx.shape
    dh = Dd // H
    queries, context = build_queries_context(ctx, ix, prm["mask_token"], prm["task_emb"], prm["pos"], mutate)
    queries.retain_grad()
    P = queries.shape[1]
    qn = rb(rf(_ln(queries, prm["query_norm_w"], prm["query_norm_b"], eps)))
    cn = rb(rf(_ln(context, prm["context_norm_w"], prm["context_norm_b"], eps)))
    q = rb(rf(qn @ rf(prm["q_w"]).t() + prm["q_b"]))
    kv = rb(rf(cn @ rf(prm["kv_w"]).t() + prm["kv_b"]))
    k, v = kv[..., :Dd], kv[..., Dd:]
    qh = q.reshape(B, P, H, dh).transpose(1, 2)
    kh = k.reshape(B, Nc, H, dh).transpose(1, 2)
    vh = v.reshape(B, Nc, H, dh).transpose(1, 2)
    o = rb(rf(attention(qh, kh, vh, 1.0 / math.sqrt(dh), round).transpose(1, 2).reshape(B, P, Dd)))
    x0 = rb(o @ rf(prm["proj_w"]).t()) + prm["proj_b"]
    h = rb(rf(_ln(x0, prm["out_norm_w"], prm["out_norm_b"], eps)))
    zp = h @ rf(prm["fc1_w"]).t() + prm["fc1_b"]
    z = rb(rf(zp))
    if fuse_gelu and round:
        # GELU in the fc1 epilogue on the fp32 pre-activation (value from zp); fc2's dgrad applies GELU'(bf16 z) to its
        # fp32 accumulator before the one bf16 store (gradient through z)
        gz = gelu(z)
        a = rf(gelu(zp).detach() + gz - gz.detach())
    else:
        # a streaming kernel applies GELU to the stored bf16 z; fc2's dgrad is stored bf16 before GELU' is applied
        a = rb(rf(gelu(z)))
    y = rf(rb(a @ rf(prm["fc2_w"]).t()) + prm["fc2_b"])
    out = x0 + y
    out.backward(dout)
    return out.detach(), queries

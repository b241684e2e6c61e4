"""Record drop_path.pt from the LIVE reference: stochastic depth in training mode.

    MULTIMAE_REFERENCE=<reference checkout> python tests/golden/make_golden_drop_path.py

A tiny3-like 3-modality MultiMAE (dim 32, encoder depth 3, decoder depth 2) built with make_golden.build_model, its
encoder and every decoder_transformer given DropPath(linspace(0, 0.5, depth)[i]) - what the constructors do with
drop_path_rate=0.5 (multimae/multimae.py, multimae/output_adapters.py: `dpr = linspace(0, drop_path_rate, depth)`);
construction consumes no random numbers for it - and one training step is run with pinned mask indices, as tiny3.pt.

The reference's DropPath modules call the module-level multimae.multimae_utils.drop_path (:105-120).  For the duration of
the run it is replaced by a wrapper that calls the original and replays its one torch.rand draw from the saved CPU
generator state to recover the keep vector floor(keep + u), checked against the original's output bit for bit.  The
reference source is not modified.  Calls are attributed to blocks in execution order: encoder blocks, then the
decoder_transformer of each output adapter in dict order; attention branch, then MLP branch.

Stored: config, state_dict, inputs, masks / index triple, drop_prob and keep vectors per block, predictions, losses and
every parameter gradient.  The recorder asserts that some block drops one sample and keeps another in both branches."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402
from make_golden import save_fixture  # noqa: E402


def _set_drop_path(MU, blocks, rate):
    dpr = [v.item() for v in torch.linspace(0, rate, len(blocks))]
    for blk, p in zip(blocks, dpr):
        blk.drop_path = MU.DropPath(p) if p > 0.0 else torch.nn.Identity()


def record_drop_path(R, name, B, size, num_encoded, seed, drop_path_rate, **kw):
    import multimae.multimae_utils as MU
    torch.manual_seed(seed)
    model = MG.build_model(R, ("rgb", "depth", "semseg"), **kw)
    _set_drop_path(MU, model.encoder, drop_path_rate)
    for ad in model.output_adapters.values():
        _set_drop_path(MU, ad.decoder_transformer, drop_path_rate)
    order = []                                     # block prefixes with p > 0, in execution order
    for i, blk in enumerate(model.encoder):
        if isinstance(blk.drop_path, MU.DropPath):
            order.append(("encoder.%d" % i, blk.drop_path.drop_prob))
    for key, ad in model.output_adapters.items():
        for i, blk in enumerate(ad.decoder_transformer):
            if isinstance(blk.drop_path, MU.DropPath):
                order.append(("output_adapters.%s.decoder_transformer.%d" % (key, i), blk.drop_path.drop_prob))
    g = torch.Generator().manual_seed(seed + 1)
    x = {"rgb": torch.randn(B, 3, size, size, generator=g), "depth": torch.randn(B, 1, size, size, generator=g),
         "semseg": torch.randint(0, 133, (B, size // 4, size // 4), generator=g)}
    torch.manual_seed(seed + 2)
    triple = model.generate_random_masks({d: torch.zeros(B, (size // 16) ** 2, 1) for d in x}, num_encoded, alphas=1.0)
    model.generate_random_masks = lambda *a, **k: triple
    calls = []
    original = MU.drop_path

    def recording_drop_path(t, drop_prob=0.0, training=False):
        if drop_prob == 0.0 or not training:
            return original(t, drop_prob, training)
        before = torch.get_rng_state()
        out = original(t, drop_prob, training)
        after = torch.get_rng_state()
        torch.set_rng_state(before)
        u = torch.rand((t.shape[0],) + (1,) * (t.ndim - 1), dtype=t.dtype, device=t.device)
        assert torch.equal(torch.get_rng_state(), after), "drop_path replay consumed a different number of draws"
        keep = (1 - drop_prob + u).floor_()
        assert torch.equal(out, t.div(1 - drop_prob) * keep), "drop_path replay diverged from the reference"
        calls.append((float(drop_prob), keep.flatten().clone()))
        return out

    MU.drop_path = recording_drop_path
    try:
        preds, masks = model(x, num_encoded_tokens=num_encoded, alphas=1.0)
        loss_fns = {"rgb": R.MSE(16, 1), "depth": R.L1(16, 1), "semseg": R.CE(16, 4),
                    "norm_rgb": R.MSE(16, 1, norm_pix=True)}
        losses = {t: loss_fns[t](preds[t].float(), x["rgb" if t == "norm_rgb" else t],
                                 mask=masks.get("rgb" if t == "norm_rgb" else t)) for t in preds}
        sum(losses.values()).backward()
    finally:
        MU.drop_path = original
    assert len(calls) == 2 * len(order), (len(calls), order)
    keep = {}
    for j, (prefix, p_) in enumerate(order):
        assert calls[2 * j][0] == calls[2 * j + 1][0] == p_, (prefix, calls[2 * j][0], p_)
        keep[prefix] = (calls[2 * j][1], calls[2 * j + 1][1])
    # the fixture must show both outcomes: some block drops one sample and keeps another in each of its two branches
    mixed = [k for k, (a, m) in keep.items() if 0 < float(a.sum()) < B and 0 < float(m.sum()) < B]
    assert mixed, {k: (a.tolist(), m.tolist()) for k, (a, m) in keep.items()}
    grads = {n: p_.grad.clone() for n, p_ in model.named_parameters() if p_.grad is not None}
    gnorm = torch.norm(torch.stack([g_.norm(2) for g_ in grads.values()]), 2)
    save_fixture({
        "config": dict(in_domains=["rgb", "depth", "semseg"], B=B, size=size, num_encoded=num_encoded, **kw,
                       drop_path_rate=drop_path_rate),
        "state_dict": {k: v.detach().clone() for k, v in model.state_dict().items()},
        "inputs": x,
        "task_masks": {k: v.clone() for k, v in masks.items()},
        "ids_keep": triple[1].clone(), "ids_restore": triple[2].clone(),
        "drop_prob": dict(order), "keep": keep,
        "preds": {k: v.detach().clone() for k, v in preds.items()},
        "losses": {k: v.detach().clone() for k, v in losses.items()},
        "grads": grads, "grad_norm": gnorm,
    }, os.path.join(HERE, name))
    print("wrote", name, {k: round(float(v), 6) for k, v in losses.items()}, "mixed blocks", mixed)


if __name__ == "__main__":
    R = MG.import_reference()
    record_drop_path(R, "drop_path.pt", B=4, size=64, num_encoded=12, seed=51, drop_path_rate=0.5, dim=32, depth=3, heads=2,
                     dec_dim=16, dec_depth=2, dec_heads=2, image_size=64)

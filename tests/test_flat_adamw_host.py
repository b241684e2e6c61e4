"""CPU: the grouped flat AdamW (multimae_b200.optim.GroupedFlatAdamW, mmae_adamw_step_groups) without a GPU.

1. The C entry point refuses every bad argument, with its message, before any launch.
2. Against a recording stub of the library: the layer-decay groups of the fine-tuning scripts (built by the stand-in
   for utils/optim_factory.py under tests/adamw_standin) cover every trainable parameter of multivit_base + a 1000-class
   head exactly once, at its arena offset, with its group's index; adjacent slots of one group form one segment; the
   lr / weight_decay in param_groups at the time of a step are what the call carries.
3. The overlay: without MMAE_FLAT_ADAMW the factory builds torch.optim.AdamW; with it, GroupedFlatAdamW - and
   torch.optim.AdamW, with one printed line, when a parameter lies outside the model.
4. state_dict round trips in both directions with torch.optim.AdamW."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from multimae_b200 import _lib as L
from multimae_b200 import functional as Fn
from multimae_b200 import optim as O
from test_drop_path_host import _Rec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STANDIN = os.path.join(ROOT, "tests", "adamw_standin")


def _factory():
    import importlib.util
    spec = importlib.util.spec_from_file_location("_standin_optim_factory",
                                                  os.path.join(STANDIN, "utils", "optim_factory.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _cls_base(seed=0):
    from multimae_b200.input_adapters import PatchedInputAdapter
    from multimae_b200.multimae import multivit_base
    from multimae_b200.output_adapters import LinearOutputAdapter
    torch.manual_seed(seed)
    return multivit_base({"rgb": PatchedInputAdapter(num_channels=3, stride_level=1, patch_size_full=16, image_size=224)},
                         {"cls": LinearOutputAdapter(1000)})


def _groups(model, weight_decay=0.05, layer_decay=0.65):
    f = _factory()
    lda = f.layer_decay_assigner(model, layer_decay)
    return f.get_parameter_groups(model, weight_decay, model.no_weight_decay(), lda.get_layer_id, lda.get_scale)


@pytest.fixture()
def rec(monkeypatch):
    r = _Rec()
    monkeypatch.setattr(L, "lib", lambda: r)
    monkeypatch.setattr(L, "current_stream", lambda: 0)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, what: None)
    monkeypatch.setattr(O, "_on_device", lambda p: True)
    return r


def _step_calls(rec):
    return [a for n, a in rec.calls if n == "mmae_adamw_step_groups"]


def test_entry_point_validates_before_any_launch():
    lib = L.lib()
    S = L.AdamwSegment
    D = ctypes.c_double * 2
    good = dict(param=256, grad=512, exp_avg=768, exp_avg_sq=1024, mirror_bf16=None, n=8, group=1, reserved=0)

    def seg(**kw):
        return (S * 2)(S(**good), S(**dict(good, **kw)))

    def call(segs=None, count=2, lr=D(1e-3, 1e-3), wd=D(0.05, 0.0), groups=2, b1=0.9, b2=0.999, eps=1e-8, step=4096):
        return lib.mmae_adamw_step_groups(seg() if segs is None else segs, count, lr, wd, groups, b1, b2, eps, None, step,
                                          None)
    before = lib.mmae_launch_count()
    nan, inf = float("nan"), float("inf")
    cases = [
        (lambda: call(segs=seg(n=-1)), b"segment 1: negative size"),
        (lambda: call(segs=seg(group=2)), b"segment 1: group 2 out of range"),
        (lambda: call(segs=seg(group=-1)), b"segment 1: group -1 out of range"),
        (lambda: call(segs=seg(param=None)), b"segment 1: null pointer"),
        (lambda: call(segs=seg(grad=None)), b"segment 1: null pointer"),
        (lambda: call(segs=seg(exp_avg=None)), b"segment 1: null pointer"),
        (lambda: call(segs=seg(exp_avg_sq=None)), b"segment 1: null pointer"),
        (lambda: call(segs=seg(exp_avg=772)), b"segment 1: pointers must be 16-byte aligned"),
        (lambda: call(segs=seg(mirror_bf16=8)), b"segment 1: pointers must be 16-byte aligned"),
        (lambda: call(lr=D(1e-3, nan)), b"group 1: non-finite lr / weight_decay"),
        (lambda: call(wd=D(inf, 0.0)), b"group 0: non-finite lr / weight_decay"),
        (lambda: call(b1=nan), b"bad betas / eps"),
        (lambda: call(b2=1.0), b"bad betas / eps"),
        (lambda: call(eps=inf), b"bad betas / eps"),
        (lambda: call(step=None), b"null step counter"),
        (lambda: call(groups=0), b"bad args"),
        (lambda: call(count=-1), b"bad args"),
        (lambda: lib.mmae_adamw_step_groups(None, 2, D(0, 0), D(0, 0), 2, 0.9, 0.999, 1e-8, None, 4096, None), b"bad args"),
        (lambda: lib.mmae_adamw_step_groups(seg(), 2, None, None, 2, 0.9, 0.999, 1e-8, None, 4096, None),
         b"null group arrays"),
    ]
    for fn, msg in cases:
        assert fn() == 1, msg
        assert msg in lib.mmae_last_error(), (msg, lib.mmae_last_error())
    # an empty segment may carry null pointers (it is skipped, as long as its group index is valid)
    assert lib.mmae_launch_count() == before
    with pytest.raises(L.MmaeError, match="group 2 out of range"):
        L.check(call(segs=seg(group=2)), "mmae_adamw_step_groups")


def test_segments_cover_every_parameter_once_with_its_group(rec):
    model = _cls_base()
    groups = _groups(model)
    assert len(groups) == 28 and sum(len(g["params"]) for g in groups) == 151
    group_of = {id(p): k for k, g in enumerate(groups) for p in g["params"]}
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    opt = O.GroupedFlatAdamW(groups, lr=1e-3, weight_decay=0.0)
    arena = opt.mmae_arena
    assert arena.owned and len(opt.param_groups) == 28
    segs = opt.segments
    # sorted, disjoint, inside the arena
    assert all(a[0] + a[1] <= b[0] for a, b in zip(segs, segs[1:]))
    assert segs[-1][0] + segs[-1][1] <= arena.flat.numel()
    # every trainable parameter: its slot inside exactly one segment, of its group; re-homed into the flat buffer
    trainable = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    assert len(trainable) == len(arena.offsets) == 151
    for n, p in trainable:
        o, numel, shape = arena.offsets[n]
        hits = [s for s in segs if s[0] <= o and o + numel <= s[0] + s[1]]
        assert len(hits) == 1 and hits[0][2] == group_of[id(p)], n
        assert p.data_ptr() == opt.flat_params.data_ptr() + 4 * o and p.grad.data_ptr() == arena.views[n].data_ptr()
        assert torch.equal(p.detach(), before[n])
    # segments hold nothing but parameter slots, and no two touching segments share a group (all merges were made)
    slots = sorted((o, (numel + 7) // 8 * 8) for o, numel, _ in arena.offsets.values())
    assert sum(s[1] for s in segs) == sum(n for _, n in slots)
    assert all(not (a[2] == b[2] and a[0] + a[1] == b[0]) for a, b in zip(segs, segs[1:]))
    runs = 1 + sum(1 for (_, p1), (_, p2) in zip(trainable, trainable[1:]) if group_of[id(p1)] != group_of[id(p2)])
    assert len(segs) == runs and len(segs) < 151
    # the table handed to the kernel
    opt.step()
    (args,) = _step_calls(rec)
    table, count, lrs, wds, ngroups, b1, b2, eps, found_inf, step, stream = args
    assert count == len(segs) and ngroups == 28 and (b1, b2, eps) == (0.9, 0.999, 1e-8) and found_inf is None
    assert step == opt._step.data_ptr() and stream == 0
    for i, (o, n, k) in enumerate(segs):
        t = table[i]
        assert (t.param, t.grad, t.exp_avg, t.exp_avg_sq, t.n, t.group) == (
            opt.flat_params.data_ptr() + 4 * o, arena.flat.data_ptr() + 4 * o, opt.exp_avg.data_ptr() + 4 * o,
            opt.exp_avg_sq.data_ptr() + 4 * o, n, k)
        assert t.mirror_bf16 is None                        # no twin off the GPU


def test_group_values_reach_the_next_call(rec):
    model = _cls_base()
    opt = O.GroupedFlatAdamW(_groups(model), lr=1e-3, weight_decay=0.0, betas=(0.9, 0.95), eps=1e-6)
    sched_lr, sched_wd = [1e-3, 5e-4, 2.5e-4], [0.05, 0.04, 0.03]
    found_inf = torch.zeros(1)
    for it in range(3):
        for g in opt.param_groups:                          # run_finetuning_cls.py:503-508
            g["lr"] = sched_lr[it] * g["lr_scale"]
            if g["weight_decay"] > 0:
                g["weight_decay"] = sched_wd[it]
        opt.fused_step(found_inf=found_inf) if it == 1 else opt.step()
        args = _step_calls(rec)[-1]
        assert list(args[2]) == [g["lr"] for g in opt.param_groups]
        assert list(args[3]) == [g["weight_decay"] for g in opt.param_groups]
        assert args[5:8] == (0.9, 0.95, 1e-6)
        assert args[8] == (found_inf.data_ptr() if it == 1 else None)
    assert sorted({w for w in _step_calls(rec)[-1][3]}) == [0.0, 0.03]
    assert [n for n, _ in rec.calls] == ["mmae_adamw_step_groups"] * 3


def test_unsupported_options_and_parameters(rec):
    model = _cls_base()
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(foreach=True), dict(foreach=False), dict(fused=True),
               dict(capturable=True)):
        with pytest.raises(NotImplementedError, match=next(iter(kw))):
            O.GroupedFlatAdamW(model.parameters(), **kw)
    stray = torch.nn.Parameter(torch.zeros(3))
    with pytest.raises(ValueError, match="not a trainable parameter"):
        O.GroupedFlatAdamW([{"params": list(model.parameters())}, {"params": [stray]}])
    opt = O.GroupedFlatAdamW(model.parameters())                 # torch's defaults, one group
    assert opt.defaults == torch.optim.AdamW([stray]).defaults
    with pytest.raises(NotImplementedError):
        opt.add_param_group({"params": [stray]})
    opt.zero_grad()
    assert not opt.mmae_arena.accumulating


def _torch_twin_state(seed, steps=3):
    """torch.optim.AdamW over the groups of an identical model, stepped with random gradients on the host."""
    model = _cls_base()
    opt = torch.optim.AdamW(_groups(model), lr=1e-3, weight_decay=0.0)
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for p in model.parameters():
            p.grad = torch.randn(p.shape, generator=g) * 1e-2
        opt.step()
    return model, opt


def test_state_dict_round_trips_with_torch_adamw(rec):
    _, stock = _torch_twin_state(5)
    sd = stock.state_dict()
    model = _cls_base()
    ours = O.GroupedFlatAdamW(_groups(model), lr=1e-3, weight_decay=0.0)
    for g in ours.param_groups:
        g["lr"] = 0.5
    ours.load_state_dict(sd)
    assert all(g["lr"] == 1e-3 for g in ours.param_groups)
    assert float(ours._step[0]) == 3.0
    params = [p for g in ours.param_groups for p in g["params"]]
    for i, p in enumerate(params):
        st = ours.state[p]
        assert torch.equal(st["exp_avg"], sd["state"][i]["exp_avg"]) and torch.equal(st["exp_avg_sq"],
                                                                                      sd["state"][i]["exp_avg_sq"])
        assert st["exp_avg"].data_ptr() - ours.exp_avg.data_ptr() == 4 * ours.mmae_arena.offsets[ours._named[i][0]][0]
    # ours -> torch: the same keys, values and per-parameter host step tensors
    back = ours.state_dict()
    assert [set(g) for g in back["param_groups"]] == [set(g) for g in sd["param_groups"]]
    assert set(back["state"]) == set(sd["state"])
    for i in sd["state"]:
        assert set(back["state"][i]) == {"step", "exp_avg", "exp_avg_sq"}
        assert back["state"][i]["step"].device.type == "cpu" and float(back["state"][i]["step"]) == 3.0
        assert back["state"][i]["step"] is not back["state"][0]["step"] or i == 0
    assert ours.state[params[0]]["step"].data_ptr() == ours._step.data_ptr()     # the live state is still the device one
    model2 = _cls_base()
    stock2 = torch.optim.AdamW(_groups(model2), lr=2e-3, weight_decay=0.0)
    stock2.load_state_dict(back)
    sd2 = stock2.state_dict()
    for i in sd["state"]:
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(sd2["state"][i][k], sd["state"][i][k]), (i, k)
    assert [{k: v for k, v in g.items() if k != "params"} for g in sd2["param_groups"]] == \
        [{k: v for k, v in g.items() if k != "params"} for g in sd["param_groups"]]
    # torch steps on from the loaded state: every step tensor advances once
    for p in model2.parameters():
        p.grad = torch.zeros_like(p)
    stock2.step()
    assert all(float(s["step"]) == 4.0 for s in stock2.state_dict()["state"].values())


# one process per run: the overlay rewires sys.modules, torch.load and DistributedDataParallel
_OVERLAY_RUN = r"""
import argparse, os, sys
import torch
sys.path.insert(0, %(root)r)
sys.path.insert(0, os.path.join(%(root)r, "tests"))
sys.path.insert(0, %(standin)r)
from multimae_b200 import _lib as L, functional as Fn, optim as O, overlay
from test_drop_path_host import _Rec
L.lib = lambda: _Rec()                        # a recording stub: no GPU here
L.current_stream = lambda: 0
Fn._require_cuda = lambda t, what: None
O._on_device = lambda p: True
overlay.install()
import utils.optim_factory as f
from test_flat_adamw_host import _cls_base
model = _cls_base()
lda = f.layer_decay_assigner(model, 0.65)
args = argparse.Namespace(opt="adamw", lr=1e-3, weight_decay=0.05, opt_eps=1e-8, opt_betas=None, momentum=0.9,
                          balancer_lr_scale=1.0)
opt = f.create_optimizer(args, model, skip_list=model.no_weight_decay(), get_num_layer=lda.get_layer_id,
                         get_layer_scale=lda.get_scale)
print("cls", type(opt).__module__ + "." + type(opt).__name__, len(opt.param_groups))
print("sgd", type(f.create_optimizer(argparse.Namespace(**dict(vars(args), opt="sgd")), torch.nn.Linear(2, 2))).__name__)
balancer = torch.nn.Module()
balancer.log_vars = torch.nn.Parameter(torch.zeros(3))
opt = f.create_optimizer(args, {"model": _cls_base(1), "balancer": balancer})
print("balancer", type(opt).__module__ + "." + type(opt).__name__)
print("ok")
"""


@pytest.mark.parametrize("switch", [None, "0", "1"])
def test_overlay_switch(switch):
    env = {k: v for k, v in os.environ.items() if k != "MMAE_FLAT_ADAMW"}
    if switch is not None:
        env["MMAE_FLAT_ADAMW"] = switch
    code = _OVERLAY_RUN % dict(root=ROOT, standin=STANDIN)
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=env)
    assert res.returncode == 0 and res.stdout.endswith("ok\n"), res.stdout + res.stderr[-3000:]
    lines = res.stdout.splitlines()
    assert "sgd SGD" in lines
    if switch == "1":
        assert "cls multimae_b200.optim.GroupedFlatAdamW 28" in lines
        fallback = [ln for ln in lines if ln.startswith("MMAE_FLAT_ADAMW:")]
        assert fallback == ["MMAE_FLAT_ADAMW: a parameter is not a trainable parameter of one MultiMAE / MultiViT model; "
                            "using torch.optim.AdamW"], lines
        assert "balancer torch.optim.adamw.AdamW" in lines
    else:
        assert "cls torch.optim.adamw.AdamW 28" in lines and "balancer torch.optim.adamw.AdamW" in lines
        assert not any(ln.startswith("MMAE_FLAT_ADAMW") for ln in lines)

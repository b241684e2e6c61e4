"""CPU: deterministic mode (torch.use_deterministic_algorithms) without a GPU.

1. The host layer keeps the library's switch equal to torch's flag and calls mmae_set_deterministic once per change;
   with the flag off, the C-ABI call sequence of a pre-training step and of a classification fine-tuning step is the
   one the host layer made before the switch existed.
2. MMAE_DETERMINISTIC=1 / warn makes the overlay set torch's flag (strict / warn_only) and CUBLAS_WORKSPACE_CONFIG.
3. The kernels added for the mode compile for sm_90a without spills, and the GEMM kernels that run with the mode off
   compile to the same SASS as before it existed.  tests/golden/gemm_sass_before_deterministic.json holds the sha256 of
   each such kernel's SASS (`_sass_digests` of the earlier gemm_wgmma.cu, built with the same nvcc flags).
"""
import json
import os
import re
import shutil
import subprocess

import pytest
import torch

from multimae_b200 import functional as Fn
from multimae_b200 import overlay
from multimae_b200.build import CSRC, NVCC_FLAGS, _nvcc
from test_host_plumbing import _inputs, stub  # noqa: F401  (fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_sass_before_deterministic.json")
# the C-ABI calls of _pretrain_step and _cls_step as the host layer made them before deterministic mode existed
# (_call_record of the earlier package's calls, recorded with the same stub)
CALL_LOG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_call_log_flag_off.json")


@pytest.fixture()
def torch_flag():
    """Restores torch's deterministic flag and the host layer's view of the library switch."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    state = Fn._deterministic
    Fn._deterministic = False
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
        Fn._deterministic = state


def _pretrain_step():
    from multimae_b200.criterion import MaskedCrossEntropyLoss, MaskedL1Loss, MaskedMSELoss
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from test_host_api import _build
    torch.manual_seed(0)
    model = _build().train()
    opt = FlatAdamW(model, lr=1e-3)
    scaler = NativeScalerWithGradNormCount(enabled=True).attach_arena(model.grad_arena())
    x = _inputs()
    preds, masks = model(x, num_encoded_tokens=12, alphas=1.0)
    fns = {"rgb": MaskedMSELoss(16, 1), "depth": MaskedL1Loss(16, 1), "semseg": MaskedCrossEntropyLoss(16, 4),
           "norm_rgb": MaskedMSELoss(16, 1, norm_pix=True)}
    loss = sum(fns[k](preds[k].float(), x["rgb" if k == "norm_rgb" else k], mask=masks["rgb" if k == "norm_rgb" else k])
               for k in preds)
    scaler(loss, opt, parameters=model.parameters())


def _cls_step():
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from test_cls_head_host import _build
    torch.manual_seed(0)
    model = _build().train()
    opt = FlatAdamW(model, lr=1e-3)
    scaler = NativeScalerWithGradNormCount(enabled=True).attach_arena(model.grad_arena())
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64)}
    loss = torch.nn.functional.cross_entropy(model(x)["cls"], torch.tensor([1, 2]))
    scaler(loss, opt, parameters=model.parameters())


def _call_record(log):
    """[name, scalar arguments] per call; shapes and flags are small here, pointers (which the allocator chooses) are not"""
    return [[n, [v for v in a if isinstance(v, (int, float)) and abs(v) < 1 << 20]] for n, a in log]


@pytest.mark.parametrize("step", [_pretrain_step, _cls_step], ids=["pretrain", "cls"])
def test_flag_off_leaves_the_call_sequence_unchanged(stub, torch_flag, step):  # noqa: F811
    torch.use_deterministic_algorithms(False)
    step()
    assert "mmae_set_deterministic" not in stub.calls
    want = json.load(open(CALL_LOG))["pretrain" if step is _pretrain_step else "cls"]
    got = _call_record(stub.log)
    assert [c[0] for c in got] == [c[0] for c in want]
    assert got == want


def test_toggling_torchs_flag_sets_the_switch_once_per_change(stub, torch_flag):  # noqa: F811
    from multimae_b200.criterion import MaskedMSELoss
    from test_cls_head_host import _build
    model = _build().train()
    x = {"rgb": torch.randn(2, 3, 64, 64), "depth": torch.randn(2, 1, 64, 64)}
    calls = lambda: stub.args_of("mmae_set_deterministic")  # noqa: E731
    model(x)
    assert calls() == []
    torch.use_deterministic_algorithms(True)
    model(x)
    model(x)
    assert calls() == [(1,)]
    torch.use_deterministic_algorithms(True, warn_only=True)   # warn_only counts as on: no change
    model(x)
    assert calls() == [(1,)]
    torch.use_deterministic_algorithms(False)
    pred, tgt = torch.randn(2, 3, 64, 64), torch.randn(2, 3, 64, 64)
    MaskedMSELoss(16, 1)(pred, tgt)                             # a stand-alone entry point notices the change
    assert calls() == [(1,), (0,)]
    torch.use_deterministic_algorithms(True, warn_only=True)
    MaskedMSELoss(16, 1)(pred, tgt)
    model(x)
    assert calls() == [(1,), (0,), (1,)]


@pytest.mark.parametrize("mode,warn", [("1", False), ("warn", True)])
def test_overlay_switch_sets_torchs_flag_and_cublas_workspace(monkeypatch, torch_flag, mode, warn):
    torch.use_deterministic_algorithms(False)
    monkeypatch.setenv("MMAE_DETERMINISTIC", mode)
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    overlay._deterministic_from_env()
    assert torch.are_deterministic_algorithms_enabled()
    assert torch.is_deterministic_algorithms_warn_only_enabled() == warn
    assert os.environ["CUBLAS_WORKSPACE_CONFIG"] == ":4096:8"
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":16:8")     # a value the user gave stays
    overlay._deterministic_from_env()
    assert os.environ["CUBLAS_WORKSPACE_CONFIG"] == ":16:8"


def test_overlay_switch_off_and_bad_values(monkeypatch, torch_flag):
    torch.use_deterministic_algorithms(False)
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    for off in (None, "0", ""):
        if off is None:
            monkeypatch.delenv("MMAE_DETERMINISTIC", raising=False)
        else:
            monkeypatch.setenv("MMAE_DETERMINISTIC", off)
        overlay._deterministic_from_env()
        assert not torch.are_deterministic_algorithms_enabled() and "CUBLAS_WORKSPACE_CONFIG" not in os.environ
    monkeypatch.setenv("MMAE_DETERMINISTIC", "yes")
    with pytest.raises(ValueError, match="MMAE_DETERMINISTIC"):
        overlay._deterministic_from_env()


# ---- what the compiler makes of the kernels ---------------------------------------------------------------------------
def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), os.path.join(os.path.dirname(_nvcc()), "cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("cuobjdump not found")


def _compile(src, out_dir):
    """sm_90a cubin of csrc/`src` with the library's nvcc flags; returns (cubin path, ptxas -v output)."""
    cubin = os.path.join(out_dir, os.path.splitext(src)[0] + ".cubin")
    flags = [f for f in NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC")]
    res = subprocess.run([_nvcc()] + flags + ["-Xptxas", "-v", "-cubin", os.path.join(CSRC, src), "-o", cubin],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return cubin, res.stderr


def _demangle(names):
    res = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    assert res.returncode == 0
    return res.stdout.split("\n")[:len(names)]


def _sass_functions(cubin):
    """{demangled name: SASS instruction text} of every kernel in the cubin, without addresses and encodings."""
    out = subprocess.run([_cuobjdump(), "-sass", cubin], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.split("\n"):
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;?\s*/\* 0x[0-9a-f]+ \*/", line)
        if cur and m:
            funcs[cur].append(m.group(1))
    names = list(funcs)
    return {d: "\n".join(funcs[n]) for n, d in zip(names, _demangle(names))}


def _gemm_key(name):
    """'gemm_bf16_kernel<128, false, false>' for the kernels that run with deterministic mode off (the ordered
    split-K form, ORD = true, is new); None for anything else."""
    m = re.search(r"gemm_bf16_kernel<([^>]*)>", name)
    if not m:
        return None
    args = [a.strip() for a in m.group(1).split(",")]
    if len(args) == 4:
        if args[3] != "false":
            return None
        args = args[:3]
    return "gemm_bf16_kernel<%s>" % ", ".join(args)


def _sass_digests(cubin):
    import hashlib
    out = {}
    for name, text in _sass_functions(cubin).items():
        key = _gemm_key(name)
        if key:
            out[key] = hashlib.sha256(text.encode()).hexdigest()
    return out


@pytest.fixture(scope="module")
def cubins(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("det_cubin"))
    return {src: _compile(src, d) for src in ("gemm_wgmma.cu", "index_ops.cu", "losses.cu")}


def _spills(ptxas_log):
    """{mangled kernel: (spill store bytes, spill load bytes)} from ptxas -v."""
    out = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", ptxas_log):
        out[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    return out


def test_new_kernels_have_no_spills(cubins):
    wanted = {"gemm_wgmma.cu": ("splitk_reduce_kernel", "gemm_bf16_kernel"),
              "index_ops.cu": ("semseg_emb_bwd_det_kernel", "embed_assemble_bwd_kernel"),
              "losses.cu": ("regr_loss_kernel", "ce_loss_kernel")}   # (unscale_norm_kernel spilled 8 bytes before)
    checked = []
    for src, names in wanted.items():
        spills = _spills(cubins[src][1])
        demangled = dict(zip(spills, _demangle(list(spills))))
        for mangled, (st, ld) in spills.items():
            d = demangled[mangled]
            if any(n + "<" in d or n + "(" in d for n in names):
                if "gemm_bf16_kernel" in d and not d.split(">")[0].endswith("true"):
                    continue                       # the ordered forms only; the others are held to their old SASS
                assert (st, ld) == (0, 0), (d, st, ld)
                checked.append(d)
    assert sum("splitk_reduce_kernel" in d for d in checked) == 1
    assert sum("gemm_bf16_kernel" in d for d in checked) == 12     # 3 tile widths x 4 operand layouts
    assert sum("semseg_emb_bwd_det_kernel" in d for d in checked) == 1


def test_existing_gemm_kernels_compile_to_the_same_sass(cubins):
    golden = json.load(open(GOLDEN))
    now = _sass_digests(cubins["gemm_wgmma.cu"][0])
    assert set(now) == set(golden)
    assert len(golden) == 12
    changed = sorted(k for k in golden if now[k] != golden[k])
    assert not changed, changed

"""One GPU: five deterministic training steps of the bench model (MultiMAE-B, bs 128) with this tree's library and with
another build of the project, which must give bitwise the same loss, gradient norm and parameters after every step.
A change to how the GEMMs schedule or store their outputs that leaves every output element's arithmetic alone passes.

    python scripts/gpu_check_gemm_bits.py --baseline-root PATH   # PATH: a built checkout of the project to compare with

Each tree runs in a subprocess of its own (one library per process); torch.use_deterministic_algorithms(True) switches
the library's deterministic mode on, so split-K sums run in a fixed order."""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 5


def run_steps(root, out_path):
    sys.path.insert(0, root)
    import torch
    import bench
    from multimae_b200.native_scaler import NativeScalerWithGradNormCount
    from multimae_b200.optim import FlatAdamW
    from multimae_b200.train_step import TrainStep

    torch.use_deterministic_algorithms(True, warn_only=True)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model, loss_fns = bench.build_model_and_losses(dev)
    opt = FlatAdamW(model, lr=1e-4 * 128 / 256, betas=(0.9, 0.95), weight_decay=0.05)
    scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
    torch.manual_seed(1234)
    batches = [{k: v.to(dev) for k, v in bench.synthetic_batch(128, i).items()} for i in range(2)]
    step = TrainStep(model, loss_fns, opt, scaler, num_encoded_tokens=98, alphas=1.0, loss_sources={"norm_rgb": "rgb"})
    rec = []
    for i in range(STEPS):
        loss, norm = step(batches[i % 2])
        torch.cuda.synchronize()
        rec.append({"loss": loss.detach().cpu(), "norm": norm.detach().cpu(),
                    "params": torch.cat([p.detach().float().flatten() for p in model.parameters()]).cpu()})
    torch.save(rec, out_path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-root", help="a built checkout of the project to compare with")
    ap.add_argument("--run", nargs=2, metavar=("ROOT", "OUT"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.run:
        run_steps(*a.run)
        return
    import torch
    with tempfile.TemporaryDirectory() as d:
        recs = {}
        for name, root in (("baseline", os.path.abspath(a.baseline_root)), ("this tree", ROOT)):
            out = os.path.join(d, name.replace(" ", "_") + ".pt")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--run", root, out], check=True, cwd=root)
            recs[name] = torch.load(out)
    ok = True
    for i, (b, n) in enumerate(zip(recs["baseline"], recs["this tree"])):
        same = {k: torch.equal(b[k], n[k]) for k in b}
        ok &= all(same.values())
        print("step %d: loss %.7f / %.7f, grad norm %.6f / %.6f, bitwise equal: %s" % (
            i, float(b["loss"]), float(n["loss"]), float(b["norm"]), float(n["norm"]), same))
    print("ALL BITWISE EQUAL" if ok else "DIFFERENT")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()

"""2+ GPUs (torchrun): one data-parallel pre-training step in deterministic mode; rank 0 saves the loss, the reduced flat
gradient and the flat parameters after the step to OUT.  Two launches from the same seeds must save the same bits
(tests/test_cuda_deterministic.py runs it twice).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29534 \\
        scripts/gpu_check_dp_deterministic.py OUT
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench  # noqa: E402
from multimae_b200.native_scaler import NativeScalerWithGradNormCount  # noqa: E402
from multimae_b200.optim import FlatAdamW  # noqa: E402
from multimae_b200.parallel import attach_data_parallel, broadcast_parameters  # noqa: E402
from multimae_b200.train_step import TrainStep  # noqa: E402

out_path = sys.argv[1]
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
torch.use_deterministic_algorithms(True, warn_only=True)   # the model's forward switches the library's mode on

torch.manual_seed(0)
model, loss_fns = bench.build_model_and_losses(dev)
broadcast_parameters(model)
opt = FlatAdamW(model, lr=1e-3, betas=(0.9, 0.95), weight_decay=0.05)
scaler = NativeScalerWithGradNormCount(enabled=False).attach_arena(model.grad_arena())
attach_data_parallel(model, scaler)
torch.manual_seed(1234 + rank)
x = {k: v.to(dev) for k, v in bench.synthetic_batch(16, 100 * rank).items()}
step = TrainStep(model, loss_fns, opt, scaler, num_encoded_tokens=98, alphas=1.0, loss_sources={"norm_rgb": "rgb"})
loss, norm = step(x)
torch.cuda.synchronize()
if rank == 0:
    torch.save({"loss": loss.detach().cpu(), "norm": norm.detach().cpu(), "grad": model.grad_arena().flat.cpu(),
                "params": opt.flat_params.cpu()}, out_path)
    print("saved", out_path, flush=True)
dist.barrier()
dist.destroy_process_group()

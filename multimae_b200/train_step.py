"""One pre-training step (run_pretraining_multimae.py:494-537) as a reusable object, optionally replayed as ONE CUDA graph.

All shapes of the step are static (the ragged Dirichlet sampling still yields exactly `num_encoded_tokens` per sample),
no kernel of the path synchronises with the host, and every buffer the C ABI sees is owned by torch's allocator, so the
whole forward + losses + backward + gradient all-reduce hooks + unscale/norm + AdamW sequence (~900 launches) can be
captured once and replayed: the host then costs one graph launch per step instead of ~900 kernel launches and ~70
autograd-function dispatches.  The only host work left per step is the Dirichlet draw (copied into a static buffer)."""
import os

import torch

from . import _lib as L


class TrainStep:
    def __init__(self, model, loss_fns, optimizer, scaler, num_encoded_tokens=98, alphas=1.0, sample_tasks_uniformly=False,
                 loss_sources=None, standardize_depth=False):
        self.model, self.loss_fns, self.opt, self.scaler = model, loss_fns, optimizer, scaler
        # truncated depth standardisation of the 'depth' entry before it is used as input AND as loss target
        # (run_pretraining_multimae.py:487-492; --standardize_depth): one radix-select kernel instead of a full sort
        self.standardize_depth = standardize_depth
        self._pdl_default = os.environ.get("MMAE_PDL", "0") != "0"
        self.num_encoded_tokens, self.alphas, self.uniform = num_encoded_tokens, alphas, sample_tasks_uniformly
        self.loss_sources = loss_sources or {}          # output key -> input key holding its target / mask
        self.graph = None
        self.static_x = None
        self.static_out = None

    # the eager step: exactly the body of train_one_epoch between the H2D copy and the optimizer step
    def _step(self, x):
        if self.standardize_depth and "depth" in x:
            from .functional import standardize_depth
            x = dict(x)
            x["depth"] = standardize_depth(x["depth"])
        preds, masks = self.model(x, num_encoded_tokens=self.num_encoded_tokens, alphas=self.alphas,
                                  sample_tasks_uniformly=self.uniform)
        task_losses = {}
        for task in preds:
            src = self.loss_sources.get(task, task)
            task_losses[task] = self.loss_fns[task](preds[task].float(), x[src], mask=masks.get(src))
        loss = sum(task_losses.values())
        self.opt.zero_grad()
        grad_norm = self.scaler(loss, self.opt, clip_grad=None, skip_grad=None, parameters=None)
        return loss.detach(), grad_norm

    def __call__(self, x, use_graph=True):
        if self.graph is None or not use_graph:
            return self._step(x)
        if self.model.external_shares is not None:       # host-side Dirichlet draw -> static device buffer
            n_tasks = len([d for d in x if d in self.model.input_adapters])
            B = next(iter(x.values())).shape[0]
            shares = self.model.draw_task_shares(B, n_tasks, self.alphas, self.uniform)
            self._shares_host.copy_(shares)
            self.model.external_shares.copy_(self._shares_host, non_blocking=True)
        for k, v in x.items():
            self.static_x[k].copy_(v, non_blocking=True)
        if hasattr(self.opt, "sync_hyperparams"):
            self.opt.sync_hyperparams()
        self.graph.replay()
        return self.static_out

    def capture(self, example_x, warmup=3):
        """Warm up eagerly (lazy kernel attributes, workspaces, arena) then capture the step into a CUDA graph.

        The learning rate and the step count live on the device and follow the schedule across replays
        (FlatAdamW.sync_hyperparams); betas, eps and the weight decay are launch arguments and therefore frozen at their
        capture-time values - with a weight-decay schedule (run_pretraining_multimae.py:479-480, off by default:
        --weight_decay_end is None) re-capture when the value changes or run the step eagerly."""
        dev = next(iter(example_x.values())).device
        n_tasks = len([d for d in example_x if d in self.model.input_adapters])
        B = next(iter(example_x.values())).shape[0]
        self.static_x = {k: v.clone() for k, v in example_x.items()}
        # Task shares: drawn on the device inside the graph (no per-step host -> device copy: a small H2D on the compute
        # stream queues behind the in-flight input-batch copy on the one H2D engine and stalls the step until it is done).
        # Sampling uniformly over task subsets keeps the reference's host draw, fed through a static buffer.
        self._shares_host = None
        self.model.external_shares = None
        self.model.device_shares = not self.uniform
        if self.uniform:
            self._shares_host = torch.empty((B, n_tasks), dtype=torch.float32).pin_memory()
            self._shares_host.copy_(self.model.draw_task_shares(B, n_tasks, self.alphas, self.uniform))
            self.model.external_shares = self._shares_host.to(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._step(self.static_x)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        # Captured nodes get plain edges: a graph's kernel-to-kernel edges are already tight, and programmatic dependent
        # launch can leave stale L1 lines for non-coherent loads (runtime.cu).
        lib = L.lib()
        lib.mmae_set_pdl(0)
        try:
            with torch.cuda.graph(graph, stream=side):   # the warm-up stream: per-stream scratch already exists
                self.static_out = self._step(self.static_x)
        finally:
            lib.mmae_set_pdl(1 if self._pdl_default else 0)
        self.graph = graph
        return self


class InputPrefetcher:
    """Double-buffered host -> device staging of input batches on a copy stream (what the reference's DataLoader with
    pin_memory + `.to(device, non_blocking=True)` does, run_pretraining_multimae.py:445-449, without per-step
    allocations): `submit(host_batch)` enqueues the H2D copies of the NEXT batch into a free device slot while the
    current step runs; `get()` hands out the oldest submitted batch once the compute stream has been told to wait for its
    copies; `release(batch)` marks the slot reusable after the kernels enqueued so far."""

    def __init__(self, example_host_batch, device, slots=2):
        self.device = device
        self.copy_stream = torch.cuda.Stream(device=device)
        self.slots = [{k: torch.empty(v.shape, dtype=v.dtype, device=device) for k, v in example_host_batch.items()}
                      for _ in range(slots)]
        self.copied = [torch.cuda.Event() for _ in range(slots)]
        self.consumed = [None] * slots
        self.queue = []
        self.next_slot = 0
        self.bytes_per_batch = sum(v.numel() * v.element_size() for v in example_host_batch.values())

    def submit(self, host_batch):
        k = self.next_slot
        self.next_slot = (k + 1) % len(self.slots)
        with torch.cuda.stream(self.copy_stream):
            if self.consumed[k] is not None:
                self.copy_stream.wait_event(self.consumed[k])      # the step that read this slot has finished with it
            for name, t in host_batch.items():
                self.slots[k][name].copy_(t, non_blocking=True)
            self.copied[k].record(self.copy_stream)
        self.queue.append(k)

    def get(self):
        k = self.queue.pop(0)
        torch.cuda.current_stream(self.device).wait_event(self.copied[k])
        return k, self.slots[k]

    def release(self, k):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self.consumed[k] = ev

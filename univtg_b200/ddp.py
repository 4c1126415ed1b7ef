"""Data-parallel training of the UniVTG path: batches shard by video-query pair, parameters stay replicated, and the only
cross-GPU exchange is ONE all-reduce (average) of the flat gradient buffer per step (reference: DDP's bucketed gradient
all-reduce, main/train_vlp_ddp.py:272-275; SURVEY.md section 2.2 row C1).

Usage (one process per GPU, torchrun):
    dist.init_process_group("nccl")
    model, criterion = build_model(args); model.to(device)
    ddp.broadcast_parameters(model)              # what the DDP constructor does (rank 0 -> all)
    ddp.attach_flat_allreduce(model)             # one NCCL all-reduce issued at the end of the fused backward
    ... the usual loop: outputs = model(**inputs); loss = ...; loss.backward(); optimizer.step()

The reference's own script wraps the model in torch DistributedDataParallel(find_unused_parameters=True); that also works
unchanged with this model (gradients reach param.grad through autograd), with DDP's 25 MB buckets instead of one buffer.
"""
import os

import torch
import torch.distributed as dist


def broadcast_parameters(model, src=0, group=None):
    """Make every rank start from rank `src`'s parameters and buffers."""
    for t in list(model.parameters()) + list(model.buffers()):
        dist.broadcast(t.data, src=src, group=group)


def make_flat_allreduce_hook(group=None):
    """Returns hook(flat): in-place average of `flat` over the process group with a single collective."""
    world = dist.get_world_size(group)
    backend = dist.get_backend(group)

    def hook(flat):
        if world == 1:
            return
        if backend == "nccl":
            dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=group)  # NVLink/NVSwitch; NVLS in-switch reduction when available
        else:
            dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
            flat.div_(world)

    return hook


def grad_stage_slices(model):
    """[(stage, [(lo, hi), ...]), ...]: slices of the flat gradient buffer that become final at each backward stage
    (univtg_backward_stages), in completion order.  Together they cover every parameter exactly once: with use_txt_pos the three
    txt_position_embed gradients appended after the C-ABI list are final at stage n - 2 (include/univtg_b200.h)."""
    import ctypes

    from . import _lib

    lib = _lib.load_library()
    cfg = model._cfgs[model._fmt(True)]
    n = lib.univtg_backward_stages(ctypes.byref(cfg), None, 0)
    if n < 0:
        raise RuntimeError("univtg_b200: " + _lib.last_error())
    arr = (ctypes.c_int32 * (4 * n))()
    if lib.univtg_backward_stages(ctypes.byref(cfg), arr, n) != n:
        raise RuntimeError("univtg_b200: " + _lib.last_error())
    offs = model._grad_offsets()  # [n_params + 1] float offsets of the 16-byte aligned views
    out = []
    for k in range(n):
        sl = []
        for j in (0, 2):
            first, last = arr[4 * k + j], arr[4 * k + j + 1]
            if last > first:
                sl.append((offs[first], offs[last]))
        if model.use_txt_pos and k == n - 2:
            sl.append((offs[-4], offs[-1]))
        out.append((k, sl))
    return out


class OverlappedGradExchange:
    """Average the flat gradient buffer over the group in `enc_layers + 3` slices, each all-reduced on a side stream as soon
    as the fused backward has finished writing it (CUDA events recorded by univtg_backward), so the NVLink traffic of the
    heads / late encoder layers overlaps the backward of the earlier layers - what DDP's bucketed all-reduce does for the
    reference (main/train_vlp_ddp.py:272-275)."""

    def __init__(self, model, group=None):
        self.group = group
        self.world = dist.get_world_size(group)
        self.backend = dist.get_backend(group)
        self.stages = grad_stage_slices(model)
        self.events = None
        self.comm_stream = None
        # SMs left to the collective's CTAs while it overlaps the backward: an NCCL CTA cannot share an SM with a GEMM CTA (registers),
        # so the reserve follows NCCL_MAX_CTAS, the cap on what NCCL takes (default 32; tools/scaling_sweep.sh sweeps it).
        default_reserve = os.environ.get("NCCL_MAX_CTAS", "32")
        self.sm_reserve = int(os.environ.get("UNIVTG_DDP_SM_RESERVE", default_reserve)) if self.backend == "nccl" else 0

    def _reduce(self, t):
        if self.backend == "nccl":
            dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
            t.div_(self.world)

    def before_backward(self, plan):
        """Install the stage events on `plan` (once per plan)."""
        import ctypes

        from . import _lib

        if self.world == 1:
            return
        if self.events is None:
            self.comm_stream = torch.cuda.Stream()
            self.events = [torch.cuda.Event() for _ in self.stages]
            for e in self.events:
                e.record()  # materialises the cudaEvent_t handle
        # the armed state lives on the plan entry itself: id(plan) of an evicted entry is recycled by CPython for the next one,
        # which would then run its backward without stage events while the exchange waits on stale, already-completed ones
        if plan.grad_events_owner is not self:
            arr = (ctypes.c_void_p * len(self.events))(*[e.cuda_event for e in self.events])
            lib = _lib.load_library()
            _lib.check(lib.univtg_plan_set_grad_events(plan.handle, arr, len(self.events)), "univtg_plan_set_grad_events")
            if getattr(self, "sm_reserve", 0) > 0:  # the all-reduce kernels hold SMs while the backward's persistent GEMM grids run
                sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
                _lib.check(lib.univtg_plan_set_backward_sm_budget(plan.handle, max(8, sms - self.sm_reserve)),
                           "univtg_plan_set_backward_sm_budget")
            plan.grad_events_owner = self

    def after_backward(self, flat):
        """All launches of the backward are enqueued: chain one all-reduce per stage behind its event."""
        if self.world == 1:
            return
        if not flat.is_cuda:  # host tensors (gloo tests): same slices, no streams
            for _, sl in self.stages:
                for lo, hi in sl:
                    self._reduce(flat[lo:hi])
            return
        main = torch.cuda.current_stream()
        with torch.cuda.stream(self.comm_stream):
            for (k, sl), ev in zip(self.stages, self.events):
                self.comm_stream.wait_event(ev)
                for lo, hi in sl:
                    self._reduce(flat[lo:hi])
        main.wait_stream(self.comm_stream)  # the optimizer (or anything else reading .grad) runs after the exchange


def attach_flat_allreduce(model, group=None, overlap=False):
    """Install the gradient exchange on a univtg_b200 model (runs inside its fused backward).
    overlap=False: ONE all-reduce of the flat buffer after the backward.
    overlap=True : the buffer is reduced in stage slices on a side stream while the backward is still running."""
    model.direct_grad = True  # gradients are handed to param.grad as views of the flat buffer (no autograd accumulation copies)
    if overlap:
        model._grad_sync = OverlappedGradExchange(model, group)
        model._flat_grad_hook = None
    else:
        model._grad_sync = None
        model._flat_grad_hook = make_flat_allreduce_hook(group)
    return model


def detach_flat_allreduce(model):
    model._flat_grad_hook = None
    model._grad_sync = None
    model.direct_grad = False
    return model

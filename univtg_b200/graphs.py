"""A training step replayed from a CUDA graph.

    from univtg_b200.graphs import GraphedTrainStep
    step = GraphedTrainStep(model, criterion, optimizer)   # optimizer: univtg_b200.optim.FlatAdamW
    for inputs, targets in loader:
        total, losses = step(inputs, targets)             # = the reference loop body (main/train_mr.py:56-66), one replay

One call is `out = model(**inputs); losses = criterion(out, targets); total = criterion.weighted_total(losses);
optimizer.zero_grad(); total.backward(); optimizer.step()` - about 120 kernel launches and their Python glue - issued as ONE
graph launch.  What the eager step fixes on the host at every step is read from device memory inside the graph instead:

  * the dropout / DropPath seed: the graph starts with univtg_rng_advance (seed = univtg_rng_seed_at(seed_base, k) at replay k)
    and the plans it replays read that seed (univtg_plan_set_seed_source), so every replay draws new masks;
  * AdamW's lr and step: univtg_adamw_step_dev reads lr from a device scalar (refreshed outside the graph when
    optimizer.lr changes, e.g. by a scheduler), reads the step from a device counter it advances only when the update was not
    skipped, and takes the bias corrections from a host-built table - bit-identical to the eager univtg_adamw_step;
  * the skip flag of the update (non-finite gradients) is copied to pinned memory inside the graph and consumed one call later,
    exactly where the eager FlatAdamW.step consumes it: a skipped update is not counted, and with dynamic loss scaling the
    scale backs off; a new grad_scale selects (or captures) another graph.

One graph per (B, Lv, Lt, input dtypes, target keys and shapes, grad_scale, dropout rates, optimizer constants), kept in an
LRU of `max_graphs`.  All graphs of one GraphedTrainStep share one training workspace and one text-position scratch (sized for
the largest shape seen) and one graph memory pool, so memory does not grow with the number of graphs.  Outputs are static:
the next call overwrites them (as with torch.cuda.graphs).  Eager steps may be mixed in freely; re-seating the parameters
(model.to(), FlatAdamW re-flattening) or optimizer.load_state_dict() drops every graph.
"""
import collections
import ctypes
import time

import torch

from . import _lib

_U64 = 0xFFFFFFFFFFFFFFFF
_FLAG_SLOTS = 4  # pinned overflow-flag ring: replay k writes slot k % 4, call k + 1 reads it


def rng_seed_at(base, k):
    """The seed replay k (k = 1, 2, ...) of a GraphedTrainStep with seed_base `base` draws its masks from."""
    return int(_lib.load_library().univtg_rng_seed_at(int(base) & _U64, int(k) & _U64))


def bias_correction_table(beta1, beta2, steps=None):
    """[steps, 2] float32 (bc1, bc2_sqrt) of AdamW steps 1 .. steps, computed by the library on the host with univtg_adamw_step's
    own expressions; steps=None: just long enough that every later step has (1.0, 1.0)."""
    lib = _lib.load_library()
    if steps is None:
        steps = lib.univtg_adamw_bias_table_len(float(beta1), float(beta2))
        if steps <= 0:
            raise ValueError(_lib.last_error())
    out = torch.empty(int(steps), 2, dtype=torch.float32)
    _lib.check(lib.univtg_adamw_bias_table(float(beta1), float(beta2), int(steps), ctypes.c_void_p(out.data_ptr())),
               "univtg_adamw_bias_table")
    return out


class _Graph:
    __slots__ = ("graph", "plan", "static_in", "static_tg", "static_tg_all", "static_mask", "total", "losses")


class GraphedTrainStep:
    """`step(inputs, targets[, mask_GT])` runs one training step of `model` / `criterion` / `optimizer` from a CUDA graph and
    returns (total, losses): the weighted total and the loss dict, static tensors the next call overwrites.  mask_GT is the
    third argument of the QFVS criterion (univtg_b200.qfvs.QFVSCriterion)."""

    def __init__(self, model, criterion, optimizer, max_graphs=8):
        from .optim import FlatAdamW

        if not isinstance(optimizer, FlatAdamW):
            raise TypeError("GraphedTrainStep: the optimizer must be univtg_b200.optim.FlatAdamW (its update runs inside the graph)")
        if optimizer.model is not model:
            raise ValueError("GraphedTrainStep: the optimizer was built for another model")
        if int(max_graphs) < 1:
            raise ValueError(f"GraphedTrainStep: max_graphs must be >= 1, got {max_graphs}")
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        self.max_graphs = int(max_graphs)
        self._refuse(at_call=False)
        dev = model._device()
        # one draw from torch's CPU generator, like the eager step's per-forward seed: reproducible under torch.manual_seed
        self.seed_base = int(torch.empty((), dtype=torch.int64).random_().item()) & _U64
        self.replays = 0  # host mirror of the device counter: replay k draws from rng_seed_at(seed_base, k)
        with torch.cuda.device(dev):
            self._counter = torch.zeros(1, dtype=torch.int64, device=dev)
            self._seed = torch.zeros(1, dtype=torch.int64, device=dev)
            self._lr = torch.zeros(1, dtype=torch.float32, device=dev)
            self._step = torch.zeros(1, dtype=torch.int32, device=dev)
            self._flags_dev = torch.zeros(_FLAG_SLOTS, dtype=torch.float32, device=dev)
            self._flags_host = torch.zeros(_FLAG_SLOTS, dtype=torch.float32).pin_memory()
            self._events = [torch.cuda.Event() for _ in range(_FLAG_SLOTS)]
            self._pool = torch.cuda.graph_pool_handle()
            self._stream = torch.cuda.Stream(device=dev)  # warm-up and capture stream
        self._lr_host = None
        self._bc = {}  # (beta1, beta2) -> (device table, rows)
        self._graphs = collections.OrderedDict()
        self._ws = self._ws_key = self._tp_scratch = None
        self._sig = None
        self._last_count = self._last_event = None
        self.captures = []  # (key, seconds) of every capture, oldest first

    # -- refusals (all raised before anything is captured) ----------------------------------------------------------------
    def _refuse(self, at_call):
        model, crit = self.model, self.criterion
        if getattr(model, "operand_format", 0) == 2:
            from .plugin import STRICT_TRAINING_REFUSAL

            raise NotImplementedError(STRICT_TRAINING_REFUSAL)
        if getattr(model, "reference_rng_order", False):
            raise NotImplementedError("GraphedTrainStep: reference_rng_order draws the masks as torch tensors on the host side of the "
                                      "step; graph replay needs the in-kernel masks (reference_rng_order = False)")
        if getattr(model, "keep_last_draw", False):
            raise NotImplementedError("GraphedTrainStep: keep_last_draw materialises explicit drop-mask tensors from the host seed; "
                                      "turn it off for graph replay")
        if getattr(model, "_grad_sync", None) is not None:
            raise NotImplementedError("GraphedTrainStep: an armed ddp.OverlappedGradExchange (NCCL inside the graph) is not "
                                      "supported; train multi-GPU with eager steps")
        if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            raise NotImplementedError("GraphedTrainStep: world size > 1 is not supported (the gradient exchange is not captured)")
        if "saliency_cls" in getattr(crit, "losses", ()):
            raise NotImplementedError("loss 'saliency_cls' ('tal' train_path) is outside the accelerated path")
        if not at_call:
            return
        if not model.training or not torch.is_grad_enabled():
            raise RuntimeError("GraphedTrainStep: the model must be in train mode with autograd enabled")
        if model.__dict__.get("_flat_grad_unstepped", False):
            raise NotImplementedError("GraphedTrainStep: gradient accumulation is not supported - a backward ran since the last "
                                      "optimizer step and a graphed step starts from a zero gradient buffer; call "
                                      "optimizer.step() or optimizer.zero_grad() first")

    # -- state that invalidates every graph ----------------------------------------------------------------------------------
    def _signature(self):
        model, opt = self.model, self.optimizer
        flat_g, _ = model._grad_buffer()
        fmt = model._fmt(True)
        return (opt._flat_p.data_ptr(), flat_g.data_ptr(), opt._m.data_ptr(), opt._v.data_ptr(), opt._scratch.data_ptr(),
                model._packed[fmt].data_ptr(), model._txt_pos_ptrs(), opt._layout_version, model._device())

    def reset(self):
        """Drop every graph (they are re-captured on demand)."""
        self._graphs.clear()
        self._ws_key = None

    def _key(self, inputs, targets, mask_GT):
        model, opt = self.model, self.optimizer
        B, Lv, _ = inputs["src_vid"].shape
        Lt = inputs["src_txt"].shape[1]
        tkeys = tuple(sorted((k, str(v.dtype), tuple(v.shape)) for k, v in targets.items() if torch.is_tensor(v)))
        mk = None if mask_GT is None else (str(mask_GT.dtype), tuple(mask_GT.shape))
        return (B, Lv, Lt, tuple(str(inputs[k].dtype) for k in ("src_txt", "src_txt_mask", "src_vid", "src_vid_mask")), tkeys, mk,
                float(model.grad_scale), float(model.input_dropout), float(model.droppath), float(model.attn_dropout),
                opt.betas, opt.eps, opt.weight_decay, opt.max_grad_norm, opt.write_clipped_grads, opt.dynamic_loss_scale)

    # -- the step ------------------------------------------------------------------------------------------------------------
    def __call__(self, inputs, targets, mask_GT=None):
        from .qfvs import QFVSCriterion

        self._refuse(at_call=True)
        if isinstance(self.criterion, QFVSCriterion) and mask_GT is None:
            raise ValueError("the QFVS criterion needs mask_GT (the kept frames of the [S, Lf] segment grid)")
        model, opt = self.model, self.optimizer
        dev = model._device()
        with torch.cuda.device(dev):
            if not opt._seated():
                opt._flatten()
            model._ensure_packed(training=True)
            sig = self._signature()
            if sig != self._sig:
                self.reset()
                self._sig = sig
                self._last_count = None  # re-read lr / step from the (possibly replaced) optimizer state
            key = self._key(inputs, targets, mask_GT)
            ent = self._graphs.get(key)
            if ent is not None and (ent.plan.handle is None or model._plans.get(ent.plan.key) is not ent.plan):
                del self._graphs[key]  # its plan was evicted or destroyed
                ent = None
            # the eager zero_grad_after_step fill of the gradient buffer: the graph's backward zero-fills it itself
            pre = model.__dict__.pop("_flat_grad_prezeroed", None)
            if pre is not None:
                torch.cuda.current_stream().wait_event(pre[1])
            self._sync_state()
            if ent is None:
                ent = self._capture(key, inputs, targets, mask_GT)
            else:
                self._graphs.move_to_end(key)
            self._prepare_ws(ent)
            for k, v in ent.static_in.items():
                v.copy_(inputs[k], non_blocking=True)
            for k, v in ent.static_tg.items():
                v.copy_(targets[k], non_blocking=True)
            if ent.static_mask is not None:
                ent.static_mask.copy_(mask_GT, non_blocking=True)
            ent.graph.replay()
            self.replays += 1
            # host mirrors, in FlatAdamW.step's order: the previous step's overflow flag (its replay or eager step finished long
            # ago), then this step
            opt._consume_overflow_flag()
            opt.step_count += 1
            slot = self.replays % _FLAG_SLOTS
            ev = self._events[slot]
            ev.record()
            opt._flag_host, opt._flag_event = self._flags_host[slot:slot + 1], ev
            self._last_count, self._last_event = opt.step_count, opt._flag_event
            opt._opt_called = True  # (what torch's step wrapper records: lr schedulers then know an update has run)
            model.__dict__["_flat_grad_dirty"] = True
            model.__dict__["_flat_grad_unstepped"] = False
        return ent.total, ent.losses

    def _sync_state(self):
        """Device lr and step from the host state when they may differ: lr changed (scheduler), or an eager step / a
        load_state_dict ran since the last replay."""
        opt = self.optimizer
        lr = opt.lr
        if lr != self._lr_host:
            self._lr.fill_(lr)
            self._lr_host = lr
        if opt.step_count != self._last_count or opt._flag_event is not self._last_event:
            self._step.fill_(opt.step_count)
            if opt._flag_event is not None and opt._flag_event is opt._flag_evt:
                # the last eager step's flag is not consumed yet: if it was skipped, step_count counts one update too many
                self._step.sub_(opt._scratch[2:3].ne(0).to(torch.int32))

    def _bias_table(self):
        b = self.optimizer.betas
        ent = self._bc.get(b)
        if ent is None:
            t = bias_correction_table(b[0], b[1])
            ent = (t.to(self.model._device()), t.shape[0])
            self._bc[b] = ent
        return ent

    def _workspace(self, plan):
        """The graphs' shared training workspace / text-position scratch, grown to the largest shape seen (growing drops the
        graphs, which baked the old buffers in)."""
        model = self.model
        lib = _lib.load_library()
        dev = model._device()
        nbytes = lib.univtg_train_workspace_bytes(ctypes.byref(model._cfg), ctypes.byref(plan.shape))
        if nbytes == 0:
            raise RuntimeError("univtg_b200: " + _lib.last_error())
        if self._ws is None or self._ws.numel() < nbytes:
            self.reset()
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        if model.use_txt_pos:
            tb = lib.univtg_txt_pos_scratch_bytes(ctypes.byref(model._cfg), ctypes.byref(plan.shape))
            if self._tp_scratch is None or self._tp_scratch.numel() < tb:
                self.reset()
                self._tp_scratch = None
                self._tp_scratch = torch.empty(tb, dtype=torch.uint8, device=dev)

    def _prepare_ws(self, ent):
        """Re-establish the zero rows of the shared workspace when the previous user had another shape."""
        if self._ws_key != ent.plan.key:
            lib = _lib.load_library()
            _lib.check(lib.univtg_prepare_workspace(ctypes.byref(self.model._cfg), ctypes.byref(ent.plan.shape), _lib.ptr(self._ws), 1,
                                                    _lib.stream_ptr()), "univtg_prepare_workspace")
            self._ws_key = ent.plan.key

    def _run_step(self, ent, update):
        model, crit, opt = self.model, self.criterion, self.optimizer
        out = model(**ent.static_in)
        if ent.static_mask is not None:
            losses = crit(out, ent.static_tg_all, ent.static_mask)
        else:
            losses = crit(out, ent.static_tg_all)
        total = crit.weighted_total(losses)
        opt.zero_grad()
        total.backward()
        if update:
            self._update()
        return total, losses

    def _update(self):
        """FlatAdamW.step with the device-resident lr / step, plus the overflow flag into the pinned ring."""
        model, opt = self.model, self.optimizer
        lib = _lib.load_library()
        flat_g, _ = model._grad_buffer()
        fmt = model._fmt(True)
        cfg = model._cfgs[fmt]
        packed = model._packed[fmt]
        bc, rows = self._bias_table()
        b1, b2 = opt.betas
        _lib.check(lib.univtg_adamw_step_dev(_lib.ptr(opt._flat_p), _lib.ptr(flat_g), _lib.ptr(opt._m), _lib.ptr(opt._v), flat_g.numel(),
                                             _lib.ptr(self._lr), b1, b2, opt.eps, opt.weight_decay, _lib.ptr(self._step),
                                             opt.max_grad_norm, int(opt.write_clipped_grads), _lib.ptr(opt._scratch),
                                             ctypes.byref(cfg), _lib.ptr(packed), _lib.ptr(bc), rows, _lib.stream_ptr()),
                   "univtg_adamw_step_dev")
        params = model._packed_params()
        arr = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        _lib.check(lib.univtg_pack_vectors(ctypes.byref(cfg), arr, len(arr), _lib.ptr(packed), _lib.stream_ptr()), "univtg_pack_vectors")
        slot = torch.remainder(self._counter, _FLAG_SLOTS)
        self._flags_dev.index_copy_(0, slot, opt._scratch[2:3])
        self._flags_host.copy_(self._flags_dev, non_blocking=True)

    def _capture(self, key, inputs, targets, mask_GT):
        model = self.model
        lib = _lib.load_library()
        dev = model._device()
        B, Lv, _ = inputs["src_vid"].shape
        Lt = inputs["src_txt"].shape[1]
        t0 = time.perf_counter()
        plan = model._get_plan(B, Lv, Lt, True)  # created outside the capture
        self._workspace(plan)
        if len(self._graphs) >= self.max_graphs:
            self._graphs.popitem(last=False)
        ent = _Graph()
        ent.plan = plan
        ent.static_in = {k: torch.empty_like(inputs[k], device=dev) for k in ("src_txt", "src_txt_mask", "src_vid", "src_vid_mask")}
        ent.static_tg = {k: torch.empty_like(v, device=dev) for k, v in targets.items() if torch.is_tensor(v)}
        ent.static_tg_all = None
        ent.static_mask = None if mask_GT is None else torch.empty_like(mask_GT, device=dev)
        for k, v in ent.static_in.items():
            v.copy_(inputs[k])
        for k, v in ent.static_tg.items():
            v.copy_(targets[k])
        if ent.static_mask is not None:
            ent.static_mask.copy_(mask_GT)
        tg_all = dict(targets)
        tg_all.update(ent.static_tg)
        ent.static_tg_all = tg_all
        self._prepare_ws(ent)
        self._bias_table()  # (host-built: before the capture)
        unstepped = model.__dict__.get("_flat_grad_unstepped", False)
        rng_state = torch.get_rng_state()  # the forwards below draw (unused) host seeds: leave torch's CPU stream as it was
        model.__dict__["_graph_train_ws"] = self._ws
        if model.use_txt_pos:
            model.__dict__["_graph_txt_pos_scratch"] = self._tp_scratch
        try:
            # warm-up outside the capture, on the capture stream (library handles, autograd's device thread, the weighted-total
            # vector): forward and backward only - the parameters and the optimizer state are not touched
            side = self._stream
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._run_step(ent, update=False)
            # the autograd anchor of the fused backward is a leaf: autograd joins the stream its gradient accumulator was made on
            # at the end of every backward, so the captured step makes its own (an accumulator from an eager step would tie
            # the capture to a stream outside it)
            model.__dict__.pop("_grad_anchor", None)
            _lib.check(lib.univtg_plan_set_seed_source(plan.handle, ctypes.c_void_p(self._seed.data_ptr())),
                       "univtg_plan_set_seed_source")
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=self._pool, stream=side):
                _lib.check(lib.univtg_rng_advance(self.seed_base, _lib.ptr(self._counter), _lib.ptr(self._seed), _lib.stream_ptr()),
                           "univtg_rng_advance")
                total, losses = self._run_step(ent, update=True)
        finally:
            if plan.handle is not None:
                lib.univtg_plan_set_seed_source(plan.handle, None)  # eager steps on this plan keep their host seed
            model.__dict__.pop("_graph_train_ws", None)
            model.__dict__.pop("_graph_txt_pos_scratch", None)
            torch.set_rng_state(rng_state)
            model.__dict__["_flat_grad_unstepped"] = unstepped
        ent.graph, ent.total, ent.losses = graph, total, losses
        self._graphs[key] = ent
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.current_stream().synchronize()
        self.captures.append((key, time.perf_counter() - t0))
        return ent

    # -- introspection -------------------------------------------------------------------------------------------------------
    @property
    def num_graphs(self):
        return len(self._graphs)

    def workspace_bytes(self):
        """Bytes of the buffers all graphs share (training workspace + text-position scratch)."""
        return sum(t.numel() for t in (self._ws, self._tp_scratch) if t is not None)

"""Parameter update of the reference's training loop, fused over one flat buffer.

The reference does, per step (main/train_vlp_ddp.py:63-68 = main/train_mr.py:61-66, optimizer from main/config.py:350):

    optimizer.zero_grad(); losses.backward()
    nn.utils.clip_grad_norm_(model.parameters(), opt.grad_clip)      # grad_clip default 0.1
    optimizer.step()                                                  # torch.optim.AdamW(lr, weight_decay=wd)

`FlatAdamW` is that sequence for a `univtg_b200.plugin.Model`: the model's parameters are re-seated as views of one flat fp32
buffer laid out like the flat gradient buffer the backward kernels write (and the DDP hook all-reduces), so clipping and AdamW
are two kernel launches (univtg_adamw_step) instead of ~90 per-parameter launches.  CUDA only - there is no CPU path.
"""
import ctypes

import torch

from . import _lib


class FlatAdamW(torch.optim.Optimizer):
    """A `torch.optim.Optimizer`: ONE parameter group whose `lr / betas / eps / weight_decay` are read at every step, so the
    reference's schedulers (`WarmupStepLR`, `StepLR`, main/config.py:309-360) drive it unchanged, and `state_dict()` /
    `load_state_dict()` speak torch.optim.AdamW's format, so `--resume_all` checkpoints (main/config.py:366-372,
    main/train_mr.py:151) move between the reference's optimizer and this one in either direction."""

    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-4, max_grad_norm=0.1,
                 write_clipped_grads=False, dynamic_loss_scale=True, growth_interval=2000, max_loss_scale=65536.0,
                 zero_grad_after_step=False):
        if getattr(model, "operand_format", 0) == 2:
            from .plugin import STRICT_TRAINING_REFUSAL

            raise NotImplementedError(STRICT_TRAINING_REFUSAL)
        self.model = model
        # zero_grad_after_step: step() ends by zero-filling the flat gradient buffer on a side stream (as if zero_grad() were called
        # right after it - the reference loop calls it before the next backward anyway, train_vlp_ddp.py:63); the fill then runs
        # under the next forward instead of in front of the next backward.  Off by default: torch leaves .grad readable after step().
        self.zero_grad_after_step = bool(zero_grad_after_step) and not write_clipped_grads
        self._zero_stream = self._zero_event = None
        self.max_grad_norm = float(max_grad_norm) if max_grad_norm is not None else 0.0
        self.write_clipped_grads = bool(write_clipped_grads)
        self.step_count = 0
        # A step whose gradients are not finite is skipped ON THE DEVICE (univtg_adamw_step), in every format; its flag is read
        # back one step later (no host synchronisation in the step) and the skipped update is taken off step_count, so the bias
        # correction, state_dict()'s 'step' and skipped_steps count real updates only.  With the dynamic loss scale of the fp16
        # backward (model.grad_scale) a skipped step also halves the scale, and `growth_interval` good steps in a row double it.
        self.dynamic_loss_scale = bool(dynamic_loss_scale) and model.operand_format == 0
        self.growth_interval, self.max_loss_scale = int(growth_interval), float(max_loss_scale)
        self.skipped_steps, self._good_streak = 0, 0
        self._flag_host, self._flag_event = None, None  # the flag the next step consumes (this optimizer's or a graph replay's)
        self._flag_buf = self._flag_evt = None            # this optimizer's own pinned flag and event
        self._layout_version = 0  # bumped when the flat buffers are re-seated or the state is replaced (captured graphs bake them)
        self._flat_p = None
        self._views = None
        self._m = self._v = self._scratch = None
        model.direct_grad = True  # gradients stay in the flat buffer; param.grad are views of it
        self._flatten()
        # the keys torch.optim.AdamW keeps in a group, so a state_dict written here loads into the reference's optimizer
        defaults = dict(lr=float(lr), betas=(float(betas[0]), float(betas[1])), eps=float(eps), weight_decay=float(weight_decay),
                        amsgrad=False, maximize=False, foreach=None, capturable=False, differentiable=False, fused=None,
                        decoupled_weight_decay=True)
        # the group lists what the reference hands its AdamW (main/config.py:345-350): every trainable parameter in
        # named_parameters() order - state_dict() numbers parameters by their position in this list.  Parameters outside the
        # C-ABI list (txt_position_embed.* unless use_txt_pos: then they sit at the end of the flat buffers and are clipped and
        # updated like the rest) receive no gradient here or there and keep no state.
        torch.optim.Optimizer.__init__(self, [{"params": [p for _, p in model.named_parameters() if p.requires_grad]}], defaults)

    # the hyper-parameters live in the (single) parameter group, where torch's lr schedulers write them
    def _group(self):
        if len(self.param_groups) != 1:
            raise RuntimeError("FlatAdamW: one parameter group (the reference builds one, main/config.py:345-350)")
        return self.param_groups[0]

    lr = property(lambda self: float(self._group()["lr"]), lambda self, v: self._group().__setitem__("lr", float(v)))
    eps = property(lambda self: float(self._group()["eps"]), lambda self, v: self._group().__setitem__("eps", float(v)))
    weight_decay = property(lambda self: float(self._group()["weight_decay"]),
                            lambda self, v: self._group().__setitem__("weight_decay", float(v)))
    betas = property(lambda self: tuple(float(b) for b in self._group()["betas"]),
                     lambda self, v: self._group().__setitem__("betas", (float(v[0]), float(v[1]))))

    def add_param_group(self, group):
        if getattr(self, "param_groups", None):
            raise RuntimeError("FlatAdamW: one parameter group (the reference builds one, main/config.py:345-350)")
        return super().add_param_group(group)

    # -- layout ---------------------------------------------------------------------------------------------------------
    def _flatten(self):
        """(Re)seat every parameter as a view of one flat buffer that mirrors Model._grad_buffer()'s offsets."""
        model = self.model
        params = model._abi_params()
        for p in params:
            if not p.requires_grad:
                raise RuntimeError("FlatAdamW: frozen parameters are not supported (the reference trains all of them)")
        dev = model._device()
        if dev.type != "cuda":
            raise RuntimeError("univtg_b200: FlatAdamW needs the model on a CUDA device (no CPU path)")
        flat_g, _ = model._grad_buffer()
        flat_p = torch.zeros_like(flat_g)
        views, off = [], 0
        with torch.no_grad():
            for p in params:
                n = p.numel()
                v = flat_p[off:off + n].view_as(p)
                v.copy_(p.data)
                p.data = v
                views.append(v)
                off += (n + 3) // 4 * 4
        keep = self._m is not None and self._m.numel() == flat_p.numel() and self._m.device == flat_p.device
        self._flat_p, self._views = flat_p, views
        self._layout_version = getattr(self, "_layout_version", 0) + 1
        if not keep:
            self._m = torch.zeros_like(flat_p)
            self._v = torch.zeros_like(flat_p)
            self._scratch = torch.zeros(2048, dtype=torch.float32, device=dev)  # UNIVTG_ADAMW_SCRATCH_FLOATS

    def _seated(self):
        ps = self.model._abi_params()  # model.to() / load_state_dict(assign=True) move every parameter: two sentinels suffice per step
        return ps[0].data_ptr() == self._views[0].data_ptr() and ps[-1].data_ptr() == self._views[-1].data_ptr()

    # -- torch.optim-like surface ---------------------------------------------------------------------------------------
    def zero_grad(self, set_to_none=True):
        """The next backward writes the flat gradient buffer from scratch (it zero-fills it itself); without a zero_grad() in
        between, further backwards accumulate into it like torch's .grad (univtg_b200/autograd.py)."""
        self.model.__dict__["_flat_grad_dirty"] = False
        self.model.__dict__["_flat_grad_unstepped"] = False
        return None  # (with zero_grad_after_step the buffer is already being cleared; the backward waits for that fill)

    @torch.no_grad()
    def step(self):
        """clip_grad_norm_(max_grad_norm) + AdamW over the flat buffers; returns the total gradient norm (device scalar)."""
        model = self.model
        if not self._seated():  # e.g. model.to(...) or load_state_dict(assign=True) replaced parameter storage
            self._flatten()
        flat_g, _ = model._grad_buffer()
        if flat_g.numel() != self._flat_p.numel():
            raise RuntimeError("FlatAdamW: gradient / parameter buffer size mismatch")
        lib = _lib.load_library()
        # Inside a torch.cuda.graph capture of the whole training step the step number is baked into the graph and the host
        # cannot wait for a flag: the skip flag is neither read nor staged there.  The update itself still skips non-finite
        # gradients on the device.
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            self._consume_overflow_flag()
        self.step_count += 1
        model.__dict__["_flat_grad_unstepped"] = False
        with torch.cuda.device(flat_g.device):
            # The update kernel also refreshes the 16-bit GEMM operand copies of the weight matrices it has just computed (the
            # packed buffer of the training format), so the next forward needs no re-packing pass over the 43 M fp32 weights;
            # only the fp32 vectors (LayerNorm terms, biases, token-type rows) are re-copied by one small launch.
            model._ensure_packed(training=True)  # allocates / fully packs once; a no-op afterwards (see below)
            fmt = model._fmt(True)
            cfg = model._cfgs[fmt]
            packed = model._packed[fmt]
            _lib.check(lib.univtg_adamw_step(_lib.ptr(self._flat_p), _lib.ptr(flat_g), _lib.ptr(self._m), _lib.ptr(self._v),
                                             flat_g.numel(), self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay,
                                             self.step_count, self.max_grad_norm, int(self.write_clipped_grads),
                                             _lib.ptr(self._scratch), ctypes.byref(cfg), _lib.ptr(packed), _lib.stream_ptr()),
                       "univtg_adamw_step")
            arr = self.__dict__.get("_ptr_array")
            if arr is None or self.__dict__.get("_ptr_array_base") != self._flat_p.data_ptr():
                params = model._packed_params()
                arr = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
                self.__dict__["_ptr_array"], self.__dict__["_ptr_array_base"] = arr, self._flat_p.data_ptr()
            _lib.check(lib.univtg_pack_vectors(ctypes.byref(cfg), arr, len(arr), _lib.ptr(packed), _lib.stream_ptr()),
                       "univtg_pack_vectors")
            # the raw-pointer update does not bump autograd's version counters, so the packed-buffer key of this format is still
            # current; a second operand format (if ever packed) is stale
            for other in list(model._packed_key):
                if other != fmt:
                    model._packed_key.pop(other)
            if self.zero_grad_after_step:
                if self._zero_stream is None:
                    self._zero_stream, self._zero_event = torch.cuda.Stream(), torch.cuda.Event()
                self._zero_stream.wait_stream(torch.cuda.current_stream())  # the update (and any exchange before it) has read the buffer
                with torch.cuda.stream(self._zero_stream):
                    flat_g.zero_()
                    self._zero_event.record()
                model.__dict__["_flat_grad_prezeroed"] = (flat_g.data_ptr(), self._zero_event)
                model.__dict__["_flat_grad_dirty"] = False
            if not capturing:
                if self._flag_buf is None:
                    self._flag_buf = torch.zeros(1, dtype=torch.float32).pin_memory()
                    self._flag_evt = torch.cuda.Event()
                self._flag_buf.copy_(self._scratch[2:3], non_blocking=True)
                self._flag_evt.record()
                self._flag_host, self._flag_event = self._flag_buf, self._flag_evt
        return self._scratch[1]

    def _consume_overflow_flag(self):
        """Outcome of the PREVIOUS step (its flag copy finished long ago: no stall): a skipped update is not counted; with the
        dynamic loss scale, back off / grow the scale."""
        if self._flag_event is None:
            return
        self._flag_event.synchronize()
        skipped = float(self._flag_host[0]) != 0.0
        self._flag_host = self._flag_event = None  # consumed once
        if skipped:
            self.step_count -= 1  # that update never happened
            self.skipped_steps += 1
        if not self.dynamic_loss_scale:
            return
        if skipped:
            self._good_streak = 0
            self.model.grad_scale = max(1.0, self.model.grad_scale * 0.5)
        else:
            self._good_streak += 1
            if self._good_streak >= self.growth_interval and self.model.grad_scale < self.max_loss_scale:
                self.model.grad_scale *= 2.0
                self._good_streak = 0

    # -- checkpoints in torch.optim.AdamW's format -----------------------------------------------------------------------
    def _offsets(self):
        offs, off = {}, 0
        for p in self.model._abi_params():
            offs[id(p)] = (off, p.numel())
            off += (p.numel() + 3) // 4 * 4
        return offs

    @torch.no_grad()
    def state_dict(self):
        """{'state': {i: {'step', 'exp_avg', 'exp_avg_sq'}}, 'param_groups': [...]} exactly as torch.optim.AdamW writes it
        (parameters numbered in group order = named_parameters() order), plus a 'loss_scale' entry torch ignores.  The last
        step's skip flag is consumed first, so a checkpoint taken right after a skipped step counts real updates only."""
        self._consume_overflow_flag()
        group = self._group()
        offs = self._offsets()
        state = {}
        if self.step_count > 0 or self.skipped_steps > 0:
            for i, p in enumerate(group["params"]):
                if id(p) not in offs:
                    continue
                off, n = offs[id(p)]
                state[i] = {"step": torch.tensor(float(self.step_count)),
                            "exp_avg": self._m[off:off + n].view_as(p).clone(),
                            "exp_avg_sq": self._v[off:off + n].view_as(p).clone()}
        g = {k: v for k, v in group.items() if k != "params"}
        g["params"] = list(range(len(group["params"])))
        return {"state": state, "param_groups": [g],
                "loss_scale": {"grad_scale": float(self.model.grad_scale), "good_streak": self._good_streak,
                               "skipped_steps": self.skipped_steps, "max_grad_norm": self.max_grad_norm}}

    @torch.no_grad()
    def load_state_dict(self, sd):
        """Accepts what state_dict() above or torch.optim.AdamW.state_dict() wrote for the same parameter list."""
        group = self._group()
        groups = sd["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != len(group["params"]):
            raise ValueError("FlatAdamW.load_state_dict: expected one parameter group of "
                             f"{len(group['params'])} parameters, got {[len(g['params']) for g in groups]}")
        if groups[0].get("amsgrad") or groups[0].get("maximize"):
            raise ValueError("FlatAdamW.load_state_dict: amsgrad / maximize checkpoints are not supported")
        if not self._seated():
            self._flatten()
        offs = self._offsets()
        self._m.zero_()
        self._v.zero_()
        steps = set()
        for key, p in zip(groups[0]["params"], group["params"]):
            st = sd["state"].get(key)
            if st is None:
                continue
            if id(p) not in offs:
                raise ValueError("FlatAdamW.load_state_dict: the checkpoint holds moments for a parameter outside the univtg path")
            off, n = offs[id(p)]
            if tuple(st["exp_avg"].shape) != tuple(p.shape):
                raise ValueError(f"FlatAdamW.load_state_dict: moment shape {tuple(st['exp_avg'].shape)} vs parameter {tuple(p.shape)}")
            self._m[off:off + n].view_as(p).copy_(st["exp_avg"])
            self._v[off:off + n].view_as(p).copy_(st["exp_avg_sq"])
            steps.add(int(float(st["step"])))
        if len(steps) > 1:
            raise ValueError(f"FlatAdamW.load_state_dict: parameters at different step counts {sorted(steps)}")
        self.step_count = steps.pop() if steps else 0
        for k, v in groups[0].items():
            if k != "params":
                group[k] = v  # lr, betas, eps, weight_decay, initial_lr (schedulers), ...
        ls = sd.get("loss_scale")
        if ls:
            self.model.grad_scale = float(ls.get("grad_scale", self.model.grad_scale))
            self._good_streak = int(ls.get("good_streak", 0))
            self.skipped_steps = int(ls.get("skipped_steps", 0))
            self.max_grad_norm = float(ls.get("max_grad_norm", self.max_grad_norm))
        self._flag_event = None  # a pending overflow flag belongs to the state that was just replaced
        self._layout_version += 1

"""Host-side mirror of the reference plugin boundary for the UniVTG hot path.

    build_model(args) -> (model, criterion)          reference model/univtg.py:409-450
    model(src_txt=, src_txt_mask=, src_vid=, src_vid_mask=) -> dict   reference model/univtg.py:105-155

Same `args` fields, same forward signature, same output-dict keys, same `state_dict` keys/shapes (reference checkpoints load
with strict=True).  PyTorch is used for parameters, device memory and streams only: all arithmetic runs in the CUDA library
behind include/univtg_b200.h (univtg_b200/_lib.py).  There is no eager / CPU fallback: without the library or a GPU the
forward raises.
"""
import ctypes
import math

import torch
from torch import nn

from . import _lib


# ------------------------------------------------------------------------------------------------------------------
# parameter containers that reproduce the reference's state_dict key names (SURVEY.md A.4)
# ------------------------------------------------------------------------------------------------------------------
class _Params(nn.Module):
    """A bag of named parameters (stands in for nn.Linear / nn.LayerNorm / nn.Conv1d / nn.Embedding key layouts)."""

    def __init__(self, **shapes):
        super().__init__()
        for name, shape in shapes.items():
            self.register_parameter(name, nn.Parameter(torch.zeros(shape)))


class _Attn(nn.Module):  # keys of nn.MultiheadAttention
    def __init__(self, d):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.zeros(3 * d, d))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d))
        self.out_proj = _Params(weight=(d, d), bias=(d,))


class _EncoderLayer(nn.Module):  # keys of TransformerEncoderLayer (transformer_encoder_droppath.py:88-106)
    def __init__(self, d, ff):
        super().__init__()
        self.self_attn = _Attn(d)
        self.linear1 = _Params(weight=(ff, d), bias=(ff,))
        self.linear2 = _Params(weight=(d, ff), bias=(d,))
        self.norm1 = _Params(weight=(d,), bias=(d,))
        self.norm2 = _Params(weight=(d,), bias=(d,))


class _Encoder(nn.Module):
    def __init__(self, d, ff, n):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(d, ff) for _ in range(n)])


class _Transformer(nn.Module):
    def __init__(self, d, ff, n, nhead):
        super().__init__()
        self.encoder = _Encoder(d, ff, n)
        self.d_model = d
        self.nhead = nhead


class _TxtPos(nn.Module):  # TrainablePositionalEncoding keys (used with --use_txt_pos; otherwise they receive no gradient)
    def __init__(self, max_q_l, d):
        super().__init__()
        self.position_embeddings = _Params(weight=(max_q_l, d))
        self.LayerNorm = _Params(weight=(d,), bias=(d,))


class _ConvHead(nn.Module):  # Conv (model/univtg.py:367-382): 3 x Conv1d(k=3)
    def __init__(self, d, out_dim):
        super().__init__()
        self.layers = nn.ModuleList([_Params(weight=(d, d, 3), bias=(d,)), _Params(weight=(d, d, 3), bias=(d,)),
                                     _Params(weight=(out_dim, d, 3), bias=(out_dim,))])


class _LinearLayer(nn.Module):  # LinearLayer (model/univtg.py:384-406): LayerNorm + Sequential(Dropout, Linear)
    def __init__(self, din, dout):
        super().__init__()
        self.LayerNorm = _Params(weight=(din,), bias=(din,))
        self.net = nn.ModuleList([nn.Identity(), _Params(weight=(dout, din), bias=(dout,))])


def _uniform_(t, bound):
    with torch.no_grad():
        t.uniform_(-bound, bound)


class _PlanEntry:
    """One (B, Lv, Lt, training) shape bucket: the C plan (shape and tile widths, pointing into the shared workspace)."""
    __slots__ = ("handle", "shape", "key", "pins", "grad_events_owner", "txt_pos_scratch")

    def __init__(self):
        self.txt_pos_scratch = None    # inference plans with learned text positions: pos_t (lives as long as the plan)
        self.handle = None
        self.shape = None
        self.key = None
        self.pins = 0                  # live autograd contexts holding this plan: a pinned plan is never evicted
        self.grad_events_owner = None  # the gradient exchange whose stage events are installed on the C plan (ddp.py)


class _WorkspaceLease:
    """A training workspace (saved activations + backward scratch) checked out of the model's pool for ONE forward; it goes back
    when the backward has run or when the autograd context is dropped without one.  Two training forwards before a backward
    (micro-batches, two views summed into one loss) therefore get two buffers instead of overwriting each other."""

    def __init__(self, pool, buf, plan):
        self.pool, self.buf, self.plan = pool, buf, plan
        plan.pins += 1

    def release(self):
        if self.buf is not None:
            self.pool.append(self.buf)
            self.buf = None
            self.plan.pins -= 1

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


STRICT_TRAINING_REFUSAL = ("operand_format='fp16x3' is an inference mode: run the forward under model.eval() or torch.no_grad(), "
                           "and train with operand_format='fp16' or 'bf16'")


class Model(nn.Module):
    """H100-native UniVTG model: the reference `Model` (model/univtg.py:51-155) behind the same interface."""

    def __init__(self, args):
        super().__init__()
        d = int(args.hidden_dim)
        self.hidden_dim = d
        self.nheads = int(args.nheads)
        self.dim_feedforward = int(args.dim_feedforward)
        self.enc_layers = int(args.enc_layers)
        self.n_input_proj = int(args.n_input_proj)
        self.txt_dim = int(args.t_feat_dim)
        self.vid_dim = int(args.v_feat_dim)
        self.input_dropout = float(args.input_dropout)
        self.droppath = float(args.droppath)
        self.attn_dropout = float(args.dropout)
        self.span_loss_type = args.span_loss_type
        self.use_txt_pos = bool(args.use_txt_pos)
        self.max_v_l = int(getattr(args, "max_v_l", 75))
        self.operand_format = {"fp16": 0, "bf16": 1, "fp16x3": 2}[getattr(args, "operand_format", "fp16")]
        self.grad_scale = float(getattr(args, "grad_scale", 1024.0 if self.operand_format == 0 else 1.0))
        if bool(getattr(args, "pre_norm", False)):
            # the reference raises AttributeError here (forward_pre is not defined, transformer_encoder_droppath.py:128-134)
            raise NotImplementedError("pre_norm is not supported by the UniVTG encoder (reference has no forward_pre)")
        if args.position_embedding not in ("v2", "sine"):
            raise ValueError(f"not supported {args.position_embedding}")
        if not 1 <= self.n_input_proj <= 3:
            raise ValueError("n_input_proj must be 1, 2 or 3")

        # registration order == reference Model.__init__ (keeps state_dict / optimizer parameter order identical)
        self.transformer = _Transformer(d, self.dim_feedforward, self.enc_layers, self.nheads)
        self.max_q_l = int(args.max_q_l)
        self.txt_position_embed = _TxtPos(self.max_q_l, d)
        self.token_type_embeddings = _Params(weight=(2, d))
        self.span_embed = _ConvHead(d, 2 if self.span_loss_type == "l1" else self.max_v_l * 2)
        self.class_embed = _ConvHead(d, 1)
        dims_t = [self.txt_dim] + [d] * 3
        dims_v = [self.vid_dim] + [d] * 3
        self.input_txt_proj = nn.ModuleList([_LinearLayer(dims_t[i], d) for i in range(self.n_input_proj)])
        self.input_vid_proj = nn.ModuleList([_LinearLayer(dims_v[i], d) for i in range(self.n_input_proj)])
        self.weightedpool = _Params(weight=(d, 1))
        self.reset_parameters()

        # One 16-bit operand format per model (a wgmma takes A and B in ONE format): fp16 by default - its 11-bit
        # significand keeps the north-star tolerance - with gradients carried under a power-of-two loss scale in backward
        # (fp16 would underflow otherwise); "bf16" needs no scaling but is 8x coarser.  "fp16x3" (inference only) stores every
        # operand as fp16 hi + lo planes and multiplies A_hi B_hi + A_lo B_hi + A_hi B_lo: it tracks an fp32 forward to ~1e-6.
        self._packed = {}
        self._packed_key = {}
        self._plans = {}
        self._dim_t = None
        self._cfgs = {
            fmt: _lib.Config(d, self.nheads, self.dim_feedforward, self.enc_layers, self.n_input_proj, self.vid_dim, self.txt_dim, fmt)
            for fmt in (0, 1, 2)}
        self._cfg = self._cfgs[self.operand_format]

    # ---- initialisation with the reference's distributions --------------------------------------------------------
    def reset_parameters(self):
        with torch.no_grad():
            for name, p in self.named_parameters():
                if name.startswith("transformer."):
                    if p.dim() > 1:  # Transformer._reset_parameters: xavier-uniform on every matrix
                        nn.init.xavier_uniform_(p)
                    elif name.endswith(("norm1.weight", "norm2.weight")):
                        p.fill_(1.0)
                    elif name.endswith(("linear1.bias", "linear2.bias")):
                        fan_in = self.hidden_dim if "linear1" in name else self.dim_feedforward
                        _uniform_(p, 1.0 / math.sqrt(fan_in))
                    else:
                        p.zero_()  # in_proj_bias, out_proj.bias, LayerNorm biases
                elif name.endswith("LayerNorm.weight"):
                    p.fill_(1.0)
                elif name.endswith("LayerNorm.bias"):
                    p.zero_()
                elif name == "token_type_embeddings.weight":
                    p.normal_(0.0, 0.02)
                elif name == "txt_position_embed.position_embeddings.weight":
                    p.normal_(0.0, 1.0)
                elif name == "weightedpool.weight":
                    nn.init.xavier_uniform_(p)
                elif p.dim() >= 2:  # nn.Linear / nn.Conv1d default: kaiming_uniform(a=sqrt(5)) == U(+-1/sqrt(fan_in))
                    fan_in = p.shape[1] * (p.shape[2] if p.dim() == 3 else 1)
                    _uniform_(p, 1.0 / math.sqrt(fan_in))
                else:  # their biases
                    owner = dict(self.named_parameters())[name[:-4] + "weight"]
                    fan_in = owner.shape[1] * (owner.shape[2] if owner.dim() == 3 else 1)
                    _uniform_(p, 1.0 / math.sqrt(fan_in))

    # ---- C-ABI plumbing -----------------------------------------------------------------------------------------------
    def _apply(self, fn, *args, **kwargs):  # .to() / .cuda() / .float(): parameter storage moves
        self.__dict__.pop("_abi_cache", None)
        return super()._apply(fn, *args, **kwargs)

    def _abi_params(self):
        """Parameters in the order include/univtg_b200.h documents for univtg_pack_weights, followed with use_txt_pos by the three
        txt_position_embed tensors (univtg_backward's appended gradients).  The list is cached: the Parameter objects of this
        module never change identity; the hot loop asks for it several times per step."""
        cached = self.__dict__.get("_abi_cache")
        if cached is not None:
            return cached
        ps = []
        for proj in (self.input_vid_proj, self.input_txt_proj):
            for layer in proj:
                ps += [layer.LayerNorm.weight, layer.LayerNorm.bias, layer.net[1].weight, layer.net[1].bias]
        ps.append(self.token_type_embeddings.weight)
        for lyr in self.transformer.encoder.layers:
            ps += [lyr.self_attn.in_proj_weight, lyr.self_attn.in_proj_bias, lyr.self_attn.out_proj.weight,
                   lyr.self_attn.out_proj.bias, lyr.linear1.weight, lyr.linear1.bias, lyr.linear2.weight, lyr.linear2.bias,
                   lyr.norm1.weight, lyr.norm1.bias, lyr.norm2.weight, lyr.norm2.bias]
        for head in (self.span_embed, self.class_embed):
            for c in head.layers:
                ps += [c.weight, c.bias]
        ps.append(self.weightedpool.weight)
        if self.use_txt_pos:
            tp = self.txt_position_embed
            ps += [tp.position_embeddings.weight, tp.LayerNorm.weight, tp.LayerNorm.bias]
        self.__dict__["_abi_cache"] = ps
        return ps

    def _packed_params(self):
        """The univtg_pack_weights prefix of _abi_params() (the text-position tensors are read as they are, never packed)."""
        ps = self._abi_params()
        return ps[:-3] if self.use_txt_pos else ps

    def _arm_txt_pos(self, plan, drop_mul=None, scratch=None):
        """Install the learned text positions on `plan` (univtg_plan_set_txt_pos) with the parameters' CURRENT storage.  Inference
        plans own their scratch; a training forward passes its own (it carries statistics to its backward)."""
        if not self.use_txt_pos:
            return
        lib = _lib.load_library()
        if scratch is None:
            nbytes = lib.univtg_txt_pos_scratch_bytes(ctypes.byref(self._cfg), ctypes.byref(plan.shape))
            if plan.txt_pos_scratch is None or plan.txt_pos_scratch.device != self._device():
                plan.txt_pos_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self._device())
            scratch = plan.txt_pos_scratch
        tp = self.txt_position_embed
        for t in (tp.position_embeddings.weight, tp.LayerNorm.weight, tp.LayerNorm.bias):
            if t.dtype != torch.float32 or not t.is_contiguous() or t.device != self._device():
                raise RuntimeError("univtg_b200: txt_position_embed parameters must be contiguous float32 tensors on the model's device")
        st = _lib.TxtPos(tp.position_embeddings.weight.data_ptr(), tp.position_embeddings.weight.shape[0],
                         tp.LayerNorm.weight.data_ptr(), tp.LayerNorm.bias.data_ptr(),
                         drop_mul.data_ptr() if drop_mul is not None else None, scratch.data_ptr())
        _lib.check(lib.univtg_plan_set_txt_pos(plan.handle, ctypes.byref(st)), "univtg_plan_set_txt_pos")

    def _txt_pos_ptrs(self):
        """Storage of the text-position tensors a captured graph has baked in (FlatAdamW re-seats parameters)."""
        if not self.use_txt_pos:
            return None
        tp = self.txt_position_embed
        return tuple(t.data_ptr() for t in (tp.position_embeddings.weight, tp.LayerNorm.weight, tp.LayerNorm.bias))

    def _device(self):
        return self.weightedpool.weight.device

    def _fmt(self, training):
        return self.operand_format  # one 16-bit format per model: fp16 (default) or bf16, in eval and in training

    def _ensure_packed(self, training=False):
        """(Re)pack the fp32 parameters into the 16-bit operand buffer of the mode's format when any parameter changed."""
        lib = _lib.load_library()
        fmt = self._fmt(training)
        cfg = self._cfgs[fmt]
        params = self._packed_params()
        dev = self._device()
        if dev.type != "cuda":
            raise RuntimeError("univtg_b200: the model must live on a CUDA device (no CPU path); call model.to('cuda')")
        key = (dev.index,) + tuple((p.data_ptr(), p._version) for p in params)
        if self._packed.get(fmt) is not None and key == self._packed_key.get(fmt):
            return
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise RuntimeError("univtg_b200: parameters must be contiguous float32 tensors")
        nbytes = lib.univtg_packed_bytes(ctypes.byref(cfg))
        if nbytes == 0:
            raise RuntimeError("univtg_b200: " + _lib.last_error())
        buf = self._packed.get(fmt)
        if buf is None or buf.device != dev or buf.numel() != nbytes:
            self._packed[fmt] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            self._drop_plans()  # plans point into the old buffer
        arr = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        _lib.check(lib.univtg_pack_weights(ctypes.byref(cfg), arr, len(params), _lib.ptr(self._packed[fmt]), _lib.stream_ptr()),
                   "univtg_pack_weights")
        self._packed_key[fmt] = key

    PLAN_CACHE = 32  # shape buckets kept (LRU); collate pads to the batch maximum, so a corpus produces many (B, Lv, Lt)

    def _drop_plans(self, keep_training=False):
        """Destroy the cached plans (they point into the packed-weight buffer and the shared workspace).
        keep_training: the shared workspace is being re-allocated - training plans never touch it (univtg_forward_train /
        univtg_backward work in a leased buffer) and may be held by live autograd contexts, so they stay."""
        lib = _lib.load_library()
        self.__dict__["_graphs"] = {}  # captured graphs reference the plans' workspaces and tensor maps
        kept = {}
        for k, e in self._plans.items():
            if keep_training and k[3] == 1:
                kept[k] = e
            elif e.handle is not None:
                lib.univtg_plan_destroy(e.handle)
                e.handle = None  # a live autograd ctx that still holds this entry fails loudly instead of using a freed plan
        self._plans = kept
        self.__dict__["_ws_owner"] = None

    def __del__(self):
        try:
            self._drop_plans()
        except Exception:
            pass

    def _shared_workspace(self, nbytes):
        """ONE inference workspace for all shape buckets, sized for the largest shape seen (grown geometrically; growing drops
        the plans, which point into the old buffer)."""
        ws = self.__dict__.get("_ws_infer")
        if ws is None or ws.device != self._device() or ws.numel() < nbytes:
            self._drop_plans(keep_training=ws is not None and ws.device == self._device())
            cap = nbytes if ws is None or ws.device != self._device() else max(nbytes, int(ws.numel() * 1.5))
            ws = torch.empty(cap, dtype=torch.uint8, device=self._device())
            self.__dict__["_ws_infer"] = ws
        return ws

    def _lease_train_ws(self, plan):
        """Check a training workspace out of the pool (univtg_b200.plugin._WorkspaceLease).  Buffers are sized for the largest
        shape seen so far and shared between shapes; a buffer that last served another shape gets its zero rows re-established
        (univtg_prepare_workspace) - no per-shape allocation and no full-buffer memset in steady state."""
        pinned = self.__dict__.get("_graph_train_ws")
        if pinned is not None:  # a CUDA-graph capture (univtg_b200.graphs): the graphs' own buffer, prepared by their owner
            return _WorkspaceLease([], pinned, plan)
        lib = _lib.load_library()
        dev = self._device()
        nbytes = lib.univtg_train_workspace_bytes(ctypes.byref(self._cfg), ctypes.byref(plan.shape))
        if nbytes == 0:
            raise RuntimeError("univtg_b200: " + _lib.last_error())
        pool = self.__dict__.setdefault("_train_pool", [])
        owners = self.__dict__.setdefault("_train_ws_shape", {})
        buf = None
        for i, cand in enumerate(pool):
            if cand.device == dev and cand.numel() >= nbytes:
                buf = pool.pop(i)
                break
        if buf is None:
            if pool:  # too small for this shape: let the allocator recycle it
                owners.pop(pool.pop().data_ptr(), None)
            grow = max([nbytes] + [int(k[1]) for k in owners.values()])
            buf = torch.empty(grow, dtype=torch.uint8, device=dev)
        key = (plan.key[:3], buf.numel())
        if owners.get(buf.data_ptr()) != key:
            _lib.check(lib.univtg_prepare_workspace(ctypes.byref(self._cfg), ctypes.byref(plan.shape), _lib.ptr(buf), 1,
                                                    _lib.stream_ptr()), "univtg_prepare_workspace")
            owners[buf.data_ptr()] = key
        return _WorkspaceLease(pool, buf, plan)

    def _grad_buffer(self):
        """One flat fp32 gradient buffer with a view per parameter (C-ABI order); also the all-reduce payload."""
        params = self._abi_params()
        buf = self.__dict__.get("_flat_grad")
        # every view starts on a 16-byte boundary (128-bit reductions / stores in the backward kernels); the padding
        # floats stay zero, so the buffer is still a valid all-reduce / clip-norm payload
        total = sum((p.numel() + 3) // 4 * 4 for p in params)
        if buf is None or buf[0].device != self._device() or buf[0].numel() != total:
            flat = torch.zeros(total, dtype=torch.float32, device=self._device())
            views, off = [], 0
            for p in params:
                views.append(flat[off:off + p.numel()].view_as(p))
                off += (p.numel() + 3) // 4 * 4
            buf = (flat, views)
            self.__dict__["_flat_grad"] = buf
        return buf

    def _grad_offsets(self):
        """Float offsets of the per-parameter views inside the flat gradient buffer, plus the total ([n_params + 1])."""
        offs, off = [], 0
        for p in self._abi_params():
            offs.append(off)
            off += (p.numel() + 3) // 4 * 4
        offs.append(off)
        return offs

    def _get_dim_t(self, dev):
        if self._dim_t is None or self._dim_t.device != dev:
            # PositionEmbeddingSine (model/position_encoding.py:72-75), evaluated with the same fp32 torch expression
            dim_t = torch.arange(self.hidden_dim, dtype=torch.float32, device=dev)
            self._dim_t = (10000 ** (2 * torch.div(dim_t, 2).int() / self.hidden_dim)).contiguous()
        return self._dim_t

    def _get_plan(self, B, Lv, Lt, training):
        """Plan of a shape bucket (LRU cache).  Inference plans share ONE workspace; before a forward the caller passes the plan
        through _activate(), which re-establishes the workspace's zero rows when the previous forward had another shape."""
        key = (B, Lv, Lt, int(training))
        e = self._plans.pop(key, None)
        if e is not None:
            self._plans[key] = e  # most recently used last
            return e
        lib = _lib.load_library()
        if len(self._plans) >= self.PLAN_CACHE:
            for old_key, old in list(self._plans.items()):  # least recently used first; never a plan a live autograd ctx holds
                if old.pins == 0:
                    del self._plans[old_key]
                    self.__dict__.get("_graphs", {}).pop(old_key[:3], None)  # a captured graph replays this plan's tensor maps
                    if self.__dict__.get("_ws_owner") is old:
                        self.__dict__["_ws_owner"] = None
                    lib.univtg_plan_destroy(old.handle)
                    old.handle = None
                    break
        dev = self._device()
        cfg = self._cfgs[self._fmt(training)]
        shp = _lib.Shape(B, Lv, Lt, int(training))
        nbytes = lib.univtg_workspace_bytes(ctypes.byref(cfg), ctypes.byref(shp))
        if nbytes == 0:
            raise RuntimeError("univtg_b200: " + _lib.last_error())
        ws = self._shared_workspace(nbytes)
        e = _PlanEntry()
        e.shape = shp
        e.key = key
        handle = ctypes.c_void_p()
        # (a training plan never touches the plan workspace: univtg_forward_train / univtg_backward work in a leased buffer)
        _lib.check(lib.univtg_plan_create(ctypes.byref(cfg), ctypes.byref(shp), _lib.ptr(self._packed[self._fmt(training)]),
                                          _lib.ptr(ws), _lib.ptr(self._get_dim_t(dev)), _lib.stream_ptr(), ctypes.byref(handle)),
                   "univtg_plan_create")
        e.handle = handle
        self._plans[key] = e
        self.__dict__["_ws_owner"] = e if not training else None  # plan_create prepared the workspace for THIS shape
        return e

    @staticmethod
    def _feature_inputs(lib, plan, src_txt, src_vid):
        """Feature tensors as the kernels read them.  16-bit features (fp16 / bf16 - the packed shards of univtg_b200/data.py) are
        consumed as they are (the first LayerNorm reads 2 bytes per element; the H2D copy of a batch halves); anything else
        becomes contiguous float32 like the reference's collate output.  Both modalities must use the same element type."""
        kinds = {torch.float16: 1, torch.bfloat16: 2}
        kt, kv = kinds.get(src_txt.dtype, 0), kinds.get(src_vid.dtype, 0)
        if kt != kv or kt == 0:
            kt = 0
            txt = src_txt.detach().to(torch.float32).contiguous()
            vid = src_vid.detach().to(torch.float32).contiguous()
        else:
            txt, vid = src_txt.detach().contiguous(), src_vid.detach().contiguous()
        _lib.check(lib.univtg_plan_set_input_format(plan.handle, kt), "univtg_plan_set_input_format")
        return txt, vid

    def _activate(self, plan):
        """The shared inference workspace is about to be used by `plan`."""
        if self.__dict__.get("_ws_owner") is not plan:
            lib = _lib.load_library()
            cfg = self._cfgs[self._fmt(False)]
            _lib.check(lib.univtg_prepare_workspace(ctypes.byref(cfg), ctypes.byref(plan.shape), _lib.ptr(self._ws_infer), 0,
                                                    _lib.stream_ptr()), "univtg_prepare_workspace")
            self.__dict__["_ws_owner"] = plan

    # ---- forward ------------------------------------------------------------------------------------------------------
    def forward(self, src_txt, src_txt_mask, src_vid, src_vid_mask, src_cls=None, src_cls_mask=None):
        """
        Args (reference model/univtg.py:105; masks are float32 or bool with 1 = valid, inputs right-padded with zeros):
            src_txt [B, Lt, Dt], src_txt_mask [B, Lt], src_vid [B, Lv, Dv], src_vid_mask [B, Lv]
        Returns dict: pred_logits [B,Lv,1], pred_spans [B,Lv,2], src_vid_mask (passthrough), vid_mem_proj [B,Lv,d],
            txt_mem_proj [B,1,d], saliency_scores [B,Lv]
        """
        if src_cls is not None:
            raise NotImplementedError("src_cls (TAL class prompts, 'tal' train_path) is outside the accelerated path")
        if self.span_loss_type != "l1":
            raise NotImplementedError  # same behaviour as the reference (model/univtg.py:138)
        if src_vid.dim() != 3 or src_txt.dim() != 3 or src_vid.shape[0] != src_txt.shape[0]:
            raise ValueError("src_vid / src_txt must be [B, L, D] with the same batch size")
        if src_vid.shape[2] != self.vid_dim or src_txt.shape[2] != self.txt_dim:
            raise ValueError(f"feature dims ({src_vid.shape[2]}, {src_txt.shape[2]}) != model ({self.vid_dim}, {self.txt_dim})")
        if self.use_txt_pos and src_txt.shape[1] > self.max_q_l:  # the reference's embedding lookup raises IndexError here
            raise ValueError(f"use_txt_pos: {src_txt.shape[1]} text tokens exceed max_q_l = {self.max_q_l} learned positions")
        dev = self._device()
        if src_vid.device != dev:
            raise RuntimeError(f"inputs on {src_vid.device}, model on {dev}")
        if dev.type != "cuda":
            raise RuntimeError("univtg_b200: the model must live on a CUDA device (no CPU path); call model.to('cuda')")
        B, Lv, _ = src_vid.shape
        Lt = src_txt.shape[1]
        if tuple(src_vid_mask.shape) != (B, Lv) or tuple(src_txt_mask.shape) != (B, Lt):
            raise ValueError("mask shapes do not match the features")
        training = self.training and torch.is_grad_enabled()
        if training and self.operand_format == 2:
            raise NotImplementedError(STRICT_TRAINING_REFUSAL)
        if training:
            from .autograd import forward_train  # backward kernels live in the same library

            return forward_train(self, src_txt, src_txt_mask, src_vid, src_vid_mask)
        if getattr(self, "use_cuda_graphs", False):
            return self._forward_graphed(src_txt, src_txt_mask, src_vid, src_vid_mask)
        return self._forward_inference(src_txt, src_txt_mask, src_vid, src_vid_mask)

    def _forward_graphed(self, src_txt, src_txt_mask, src_vid, src_vid_mask):
        """Inference forward replayed from a CUDA graph (one per input shape): the ~41 kernel launches of a forward are
        captured once on static input buffers; each call copies the inputs in, replays, and returns fresh output tensors."""
        dev = self._device()
        B, Lv, _ = src_vid.shape
        Lt = src_txt.shape[1]
        key = (B, Lv, Lt)
        cache = self.__dict__.setdefault("_graphs", {})
        with torch.cuda.device(dev):
            self._ensure_packed()
            cache = self.__dict__.setdefault("_graphs", {})  # _ensure_packed may have dropped plans + graphs
            ent = cache.get(key)
            if ent is not None and ent["txt_pos"] != self._txt_pos_ptrs():
                del cache[key]  # the graph baked in text-position tensors that have been re-seated since
                ent = None
            if ent is None:
                if len(cache) >= 4:
                    cache.pop(next(iter(cache)))
                static = {"src_txt": torch.zeros(B, Lt, self.txt_dim, device=dev), "src_txt_mask": torch.zeros(B, Lt, device=dev),
                          "src_vid": torch.zeros(B, Lv, self.vid_dim, device=dev), "src_vid_mask": torch.zeros(B, Lv, device=dev)}
                for k, v in (("src_txt", src_txt), ("src_txt_mask", src_txt_mask), ("src_vid", src_vid), ("src_vid_mask", src_vid_mask)):
                    static[k].copy_(v)
                side = torch.cuda.Stream(device=dev)
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for _ in range(2):  # warm-up outside capture (plans, function attributes, allocator)
                        self._forward_inference(**static)
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    outs = self._forward_inference(**static)
                ent = {"graph": graph, "static": static, "outs": outs, "txt_pos": self._txt_pos_ptrs()}
                cache[key] = ent
            st = ent["static"]
            st["src_txt"].copy_(src_txt, non_blocking=True)
            st["src_txt_mask"].copy_(src_txt_mask, non_blocking=True)
            st["src_vid"].copy_(src_vid, non_blocking=True)
            st["src_vid_mask"].copy_(src_vid_mask, non_blocking=True)
            ent["graph"].replay()
            o = ent["outs"]
            return {"pred_logits": o["pred_logits"].clone(), "pred_spans": o["pred_spans"].clone(), "src_vid_mask": src_vid_mask,
                    "vid_mem_proj": o["vid_mem_proj"].clone(), "txt_mem_proj": o["txt_mem_proj"].clone(),
                    "saliency_scores": o["saliency_scores"].clone()}

    def _forward_inference(self, src_txt, src_txt_mask, src_vid, src_vid_mask, droppath_scale=None):
        lib = _lib.load_library()
        dev = self._device()
        B, Lv, _ = src_vid.shape
        Lt = src_txt.shape[1]
        d = self.hidden_dim
        with torch.cuda.device(dev):
            self._ensure_packed()
            plan = self._get_plan(B, Lv, Lt, False)
            self._activate(plan)
            self._arm_txt_pos(plan)
            txt, vid = self._feature_inputs(lib, plan, src_txt, src_vid)
            tmask = src_txt_mask.detach().to(torch.float32).contiguous()
            vmask = src_vid_mask.detach().to(torch.float32).contiguous()
            pred_logits = torch.empty(B, Lv, 1, device=dev)
            pred_spans = torch.empty(B, Lv, 2, device=dev)
            vid_mem_proj = torch.empty(B, Lv, d, device=dev)
            txt_mem_proj = torch.empty(B, 1, d, device=dev)
            saliency = torch.empty(B, Lv, device=dev)
            _lib.check(lib.univtg_forward(plan.handle, _lib.ptr(txt), _lib.ptr(tmask), _lib.ptr(vid), _lib.ptr(vmask),
                                          _lib.ptr(droppath_scale), _lib.ptr(pred_logits), _lib.ptr(pred_spans),
                                          _lib.ptr(vid_mem_proj), _lib.ptr(txt_mem_proj), _lib.ptr(saliency), _lib.stream_ptr()),
                       "univtg_forward")
        return {"pred_logits": pred_logits, "pred_spans": pred_spans, "src_vid_mask": src_vid_mask,
                "vid_mem_proj": vid_mem_proj, "txt_mem_proj": txt_mem_proj, "saliency_scores": saliency}

    def profile_forward(self, inputs):
        """Run one inference forward with the per-launch CUDA-event timeline on; returns [(kind, ms), ...]
        (kind 0 = row kernel, 1 = tensor-core GEMM, 2 = attention)."""
        lib = _lib.load_library()
        B, Lv, _ = inputs["src_vid"].shape
        Lt = inputs["src_txt"].shape[1]
        with torch.cuda.device(self._device()):
            self._ensure_packed()
            plan = self._get_plan(B, Lv, Lt, False)
            self._activate(plan)
            lib.univtg_plan_set_profiling(plan.handle, 1)
            try:
                self._forward_inference(**inputs)
                ms = (ctypes.c_float * 160)()
                kinds = (ctypes.c_int32 * 160)()
                n = lib.univtg_plan_read_profile(plan.handle, ms, kinds, 160)
            finally:
                lib.univtg_plan_set_profiling(plan.handle, 0)
        if n < 0:
            raise RuntimeError("univtg_b200: " + _lib.last_error())
        return [(int(kinds[i]), float(ms[i])) for i in range(n)]

    def profile_train_step(self, B, Lv, Lt, run):
        """CUDA-event timeline of ONE training step of shape (B, Lv, Lt): `run()` must execute forward + criterion + backward.
        Returns [(kind, ms), ...]: kind 0 = one row kernel of the forward, 1 = one tensor-core GEMM launch, 2 = one attention launch
        (forward or backward), 3 = whatever else ran before a backward GEMM / attention launch (row kernels, criterion, launch gaps)."""
        lib = _lib.load_library()
        with torch.cuda.device(self._device()):
            self._ensure_packed(training=True)
            plan = self._get_plan(B, Lv, Lt, True)
            lib.univtg_plan_set_profiling(plan.handle, 1)
            try:
                run()
                cap = 640
                ms = (ctypes.c_float * cap)()
                kinds = (ctypes.c_int32 * cap)()
                n = lib.univtg_plan_read_profile(plan.handle, ms, kinds, cap)
            finally:
                lib.univtg_plan_set_profiling(plan.handle, 0)
        if n < 0:
            raise RuntimeError("univtg_b200: " + _lib.last_error())
        return [(int(kinds[i]), float(ms[i])) for i in range(n)]

    def num_forward_launches(self, B, Lv, Lt):
        lib = _lib.load_library()
        with torch.cuda.device(self._device()):
            self._ensure_packed()
            plan = self._get_plan(B, Lv, Lt, False)
            self._arm_txt_pos(plan)
            return int(lib.univtg_forward_num_launches(plan.handle))


def build_model(args):
    """Same contract as reference model/univtg.py:409-450: returns (model, criterion); reads the same `args` fields."""
    from .criterion import SetCriterion

    try:
        device = torch.device(args.device)  # reference: torch.device(args.device); criterion.to(device)
    except (TypeError, RuntimeError):
        device = None
    model = Model(args)
    weight_dict = {"loss_b": args.b_loss_coef, "loss_g": args.g_loss_coef, "loss_f": args.f_loss_coef,
                   "loss_s_intra": args.s_loss_intra_coef, "loss_s_inter": args.s_loss_inter_coef}
    if args.dset_type in ["mr", "vlp"]:
        if "tal" not in args.train_path:
            losses = ["spans", "labels", "saliency"]
        else:
            losses = ["spans", "labels", "saliency_cls"]
    elif args.dset_type in ["hl", "vs"]:
        losses = ["labels", "saliency"]
    else:
        raise ValueError(f"unknown dset_type {args.dset_type}")
    criterion = SetCriterion(weight_dict=weight_dict, losses=losses, eos_coef=args.eos_coef, temperature=args.temperature,
                             span_loss_type=args.span_loss_type, max_v_l=args.max_v_l, saliency_margin=args.saliency_margin)
    if device is not None:
        criterion.to(device)
    return model, criterion

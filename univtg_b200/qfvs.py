"""Query-focused video summarisation (QFVS): the reference's `univtg_qfvs` model plugin (model/univtg_qfvs.py), which
main/train_qfvs.py and main/inference_qfvs.py load through the usual `model_id` lookup.

    from univtg_b200.qfvs import build_model
    model, criterion = build_model(args)
    loss_dict = criterion(outputs, targets, mask_GT)

The model is the MR/HL `Model` (the reference's QFVS model has the same parameters, state_dict keys and forward); only the
criterion differs.  Its losses run in the CUDA library (univtg_qfvs_loss_forward / univtg_qfvs_loss_backward) without a host
synchronisation, where the reference's masked_select, count slice and zero-sum branches synchronise four times per call.

calculate_semantic_matching (bottom of this module) is the drop-in for eval/qfvs.py's evaluation of one oracle summary.
"""
import json
import os

import numpy as np
import torch

from . import _lib
from .criterion import SetCriterion
from .losses import LossDict


class _QFVSLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred_logits, vid_mem_proj, txt_mem_proj, vmask, mask_gt, sal, has_pos, temperature):
        lib = _lib.load_library()
        dev = pred_logits.device
        B, Lv, d = vid_mem_proj.shape
        with torch.cuda.device(dev):
            pl = pred_logits.detach().to(torch.float32).contiguous()
            xv = vid_mem_proj.detach().to(torch.float32).contiguous()
            xt = txt_mem_proj.detach().to(torch.float32).contiguous()
            scratch = torch.empty(lib.univtg_loss_scratch_bytes(B, Lv), dtype=torch.uint8, device=dev)
            losses = torch.zeros(5, device=dev)
            _lib.check(lib.univtg_qfvs_loss_forward(_lib.ptr(pl), _lib.ptr(xv), _lib.ptr(xt), _lib.ptr(vmask), _lib.ptr(mask_gt),
                                                    _lib.ptr(sal), int(has_pos), B, Lv, d, float(temperature), _lib.ptr(losses),
                                                    _lib.ptr(scratch), _lib.stream_ptr()), "univtg_qfvs_loss_forward")
        ctx.saved = (xv, xt, scratch, B, Lv, d)
        return losses

    @staticmethod
    def backward(ctx, g_losses):
        lib = _lib.load_library()
        xv, xt, scratch, B, Lv, d = ctx.saved
        dev = xv.device
        with torch.cuda.device(dev):
            w = g_losses.detach().to(torch.float32).contiguous()
            d_logits = torch.empty(B, Lv, 1, device=dev)
            d_xv = torch.empty(B, Lv, d, device=dev)
            d_xt = torch.empty(B, 1, d, device=dev)
            _lib.check(lib.univtg_qfvs_loss_backward(_lib.ptr(w), _lib.ptr(xv), _lib.ptr(xt), B, Lv, d, _lib.ptr(scratch),
                                                     _lib.ptr(d_logits), _lib.ptr(d_xv), _lib.ptr(d_xt), _lib.stream_ptr()),
                       "univtg_qfvs_loss_backward")
        return d_logits, d_xv, d_xt, None, None, None, None, None


class QFVSCriterion(SetCriterion):
    """SetCriterion of model/univtg_qfvs.py (:156-377) behind the same interface."""

    def forward(self, outputs, targets, mask_GT=None):
        """Returns the reference's loss dict for one forward over S segments of Lf frames (model/univtg_qfvs.py:358-377).

        outputs: the model's dict (pred_logits [S, Lf, 1], vid_mem_proj, txt_mem_proj, src_vid_mask).
        targets: saliency_scores [1, >= S*Lf] (row 0 pairs, in order, with the kept positions), optionally saliency_pos_labels.
        mask_GT: S*Lf bools (the reference passes [1, S*Lf]); flat position i of [S, Lf] is kept iff mask_GT is set there.

        Every entry is a tensor: where the reference returns the Python float 0. (loss_s_inter always; loss_f and loss_s_intra
        when the kept targets sum to 0; loss_s_intra without saliency_pos_labels) this returns a 0 tensor whose gradient is 0.
        The losses are differentiable w.r.t. pred_logits, vid_mem_proj and txt_mem_proj; loss_s_intra is computed from the
        latter two as the model computes saliency_scores, so it is the same function of them.

        Unlike the reference, outputs["pred_logits"], outputs["saliency_scores"] and targets["saliency_scores"] are left as
        they are instead of being replaced with their masked selections; neither QFVS loop reads them afterwards.

        Raises ValueError, before anything runs on the device, for a missing or mis-sized mask_GT, a target row shorter than
        S*Lf, and a loss list with 'spans' (dset_type mr / vlp: QFVS targets carry no timestamps)."""
        if "spans" in self.losses:
            raise ValueError("the QFVS criterion has no 'spans' loss (QFVS targets carry no timestamp): use dset_type 'vs' or 'hl'")
        if mask_GT is None:
            raise ValueError("the QFVS criterion needs mask_GT (the kept frames of the [S, Lf] segment grid)")
        pl = outputs["pred_logits"]
        xv, xt = outputs["vid_mem_proj"], outputs["txt_mem_proj"]
        B, Lv = pl.shape[:2]
        n = B * Lv
        if pl.numel() != n or tuple(xv.shape[:2]) != (B, Lv) or xt.numel() != B * xv.shape[2]:
            raise ValueError(f"outputs must be pred_logits [S, Lf, 1], vid_mem_proj [S, Lf, d], txt_mem_proj [S, 1, d]; got "
                             f"{list(pl.shape)}, {list(xv.shape)}, {list(xt.shape)}")
        if mask_GT.numel() != n:
            raise ValueError(f"mask_GT has {mask_GT.numel()} elements, the outputs {n} = {B} x {Lv} positions")
        vmask = outputs["src_vid_mask"]
        if vmask.numel() != n:
            raise ValueError(f"outputs['src_vid_mask'] has {vmask.numel()} elements, expected {n}")
        ts = targets["saliency_scores"]
        if ts.dim() != 2 or ts.shape[0] < 1 or ts.shape[1] < n:
            raise ValueError(f"targets['saliency_scores'] must be [1, >= {n}] (row 0 pairs with the kept positions), got "
                             f"{list(ts.shape)}")
        dev = pl.device
        if dev.type != "cuda":
            raise RuntimeError("univtg_b200: the criterion runs on CUDA tensors only (no CPU path)")
        mask = mask_GT.detach().reshape(-1).to(device=dev, dtype=torch.bool).contiguous()
        sal = ts.detach()[0, :n].to(device=dev, dtype=torch.float32).contiguous()
        vm = vmask.detach().to(device=dev, dtype=torch.float32).contiguous()
        has_pos = "saliency" in self.losses and "saliency_pos_labels" in targets
        losses = _QFVSLossFunction.apply(pl, xv, xt, vm, mask, sal, has_pos, self.temperature)
        out = LossDict()
        out.vector = losses  # [loss_b, loss_g, loss_f, loss_s_inter, loss_s_intra] (SetCriterion.weighted_total)
        if "labels" in self.losses:
            out["loss_f"] = losses[2]
        if "saliency" in self.losses:
            out["loss_s_inter"] = losses[3]
            out["loss_s_intra"] = losses[4]
        return out


def build_model(args):
    """Same contract as reference model/univtg_qfvs.py build_model: (Model(args), QFVSCriterion); reads the same `args` fields."""
    from .plugin import build_model as _build

    model, crit = _build(args)
    qcrit = QFVSCriterion(weight_dict=crit.weight_dict, losses=crit.losses, eos_coef=crit.eos_coef, temperature=args.temperature,
                          span_loss_type=crit.span_loss_type, max_v_l=crit.max_v_l, saliency_margin=crit.saliency_margin)
    return model, qcrit.to(crit.empty_weight.device)


# ---- semantic evaluation: eval/qfvs.py calculate_semantic_matching ----------------------------------------------------------
MAX_SIDE = 1024  # shots per summary
MAX_TAGS = 64    # tag columns (Tags.mat has 48)


def tag_masks(rows):
    """Shot-tag rows [n, <= 64] of 0 / 1 -> n uint64 masks (bit c = tag column c)."""
    t = np.asarray(rows)
    if t.ndim != 2:
        raise ValueError(f"semantic matching: the selected tag rows must form a matrix, got shape {list(t.shape)}")
    if t.shape[1] > MAX_TAGS:
        raise ValueError(f"semantic matching: more than {MAX_TAGS} tag columns")
    if not np.isin(t, (0, 1)).all():
        raise ValueError("semantic matching: tags must be 0 or 1")
    bits = np.packbits(t.astype(bool), axis=1, bitorder="little")
    out = np.zeros((len(t), 8), dtype=np.uint8)
    out[:, :bits.shape[1]] = bits
    return out.view("<u8").reshape(-1)


def match_sums(pairs):
    """univtg_qfvs_match on [(machine masks, gt masks), ...] (each 1..1024 uint64 masks) -> total matched weight per pair."""
    sides = [len(x) for p in pairs for x in p]
    if min(sides) < 1 or max(sides) > MAX_SIDE:
        raise ValueError(f"semantic matching: each summary must hold 1..{MAX_SIDE} shots")
    if not torch.cuda.is_available():
        raise RuntimeError("univtg_b200: calculate_semantic_matching runs on CUDA only (no CPU path)")
    lib = _lib.load_library()
    a = np.concatenate([p[0] for p in pairs]).astype(np.uint64)
    b = np.concatenate([p[1] for p in pairs]).astype(np.uint64)
    a_off = np.concatenate([[0], np.cumsum([len(p[0]) for p in pairs])]).astype(np.int32)
    b_off = np.concatenate([[0], np.cumsum([len(p[1]) for p in pairs])]).astype(np.int32)
    host = np.concatenate([x.view(np.uint8) for x in (a, b, a_off, b_off)])
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        buf = torch.from_numpy(host).to(dev)
        s = torch.empty(len(pairs), dtype=torch.float64, device=dev)
        base = buf.data_ptr()
        oa, ob = 0, a.nbytes
        oao = ob + b.nbytes
        obo = oao + a_off.nbytes
        _lib.check(lib.univtg_qfvs_match(_lib.c_void_p(base + oa), _lib.c_void_p(base + oao), _lib.c_void_p(base + ob),
                                         _lib.c_void_p(base + obo), len(pairs), max(sides), _lib.ptr(s), _lib.stream_ptr()),
                   "univtg_qfvs_match")
        return s.cpu().numpy()


def calculate_semantic_matching(machine_summary, gt_summary, video_shots_tag, video_id):
    """eval/qfvs.py calculate_semantic_matching on the device; same arguments, same (precision, recall, f1) of np.float64.

    machine_summary / gt_summary: shot indices into video_shots_tag[video_id] (a [shots, tags] 0 / 1 matrix, as
    load_videos_tag returns), indexed with numpy's rules; machine_summary may be the CUDA `top_index` of score.topk as it is.
    The weight of a (machine, gt) pair is the semantic IoU of their tag sets; the total weight s of a maximum-weight matching
    comes from univtg_qfvs_match, then p = s / len(machine), r = s / len(gt), f1 = 2*p*r/(p+r) in numpy scalars as the reference
    computes them.  The reference adds the matched weights in networkx's set order, which depends on the string hash seed, so
    s agrees with it to the last bits only.  All weights 0 gives (0.0, 0.0, nan), as in the reference.

    Raises, before any launch: IndexError for an index outside the tag rows, ValueError for an empty summary (the reference's
    scikit-learn error), non-binary tags, more than 64 tag columns or more than 1,024 shots in a summary.  CUDA only."""
    tags = np.asarray(video_shots_tag[video_id])
    if torch.is_tensor(machine_summary):
        machine_summary = machine_summary.cpu().numpy()
    a_rows, b_rows = tags[machine_summary], tags[gt_summary]
    for rows, what in ((a_rows, "machine"), (b_rows, "ground-truth")):
        _check_not_empty(rows, what)
    a, b = tag_masks(a_rows), tag_masks(b_rows)
    return precision_recall_f1(np.float64(match_sums([(a, b)])[0]), a_rows.shape[0], b_rows.shape[0])


def _check_not_empty(rows, what):
    if rows.ndim == 2 and rows.shape[0] == 0:
        raise ValueError(f"Found array with 0 sample(s) (shape={rows.shape}) while a minimum of 1 is required: empty {what} summary")


def precision_recall_f1(s, n_machine, n_gt):
    """The tail of calculate_semantic_matching: numpy scalars from the matched weight s (np.float64) and the two summary sizes."""
    precision = s / n_machine
    recall = s / n_gt
    f1 = 2 * precision * recall / (precision + recall)
    return precision, recall, f1


# ---- evaluation epoch: main/inference_qfvs.py / main/train_qfvs.py eval_epoch -------------------------------------------
SUMMARY_DIR = "./data/qfvs/metadata/origin_data/Query-Focused_Summaries/Oracle_Summaries/P0"
TRANSFER = {"Cupglass": "Glass", "Musicalinstrument": "Instrument", "Petsanimal": "Animal"}
SELECT_MAX_N = 8192      # kept positions per query (one shared-memory sort); the default 20 x 200 grid keeps at most 4,000
ROWS_PER_FORWARD = 200   # samples (segments) per batched forward: 10 query files at max_segment_num = 20


def load_videos_tag(mat_path):
    """eval/qfvs.py load_videos_tag: Tags.mat -> one [shots, tags] array per video (entry [0][0] of each shot cell)."""
    import scipy.io

    mat = scipy.io.loadmat(mat_path)
    return [np.array([shot[0][0] for shot in video[0]]) for video in mat["Tags"][0]]


def l2_normalize_np_array(x, eps=1e-5):  # utils/basic_utils.py
    return x / (np.linalg.norm(x, axis=-1, keepdims=True) + eps)


def output_type(opt, config):
    """The reference's choice: 0 = pred_logits, 1 = saliency_scores, 2 = their sum (qfvs_score_ensemble)."""
    if opt.f_loss_coef == 0:
        return 1
    if opt.s_loss_intra_coef == 0:
        return 0
    return 2 if config["qfvs_score_ensemble"] > 0 else 0


def _model_device(model):
    for t in list(model.parameters()) + list(model.buffers()):
        return t.device
    return torch.device("cpu")


def _pinned(host_bytes, dev):
    """uint8 numpy -> device tensor through pinned staging (the copy does not synchronise the stream)."""
    return torch.from_numpy(host_bytes).pin_memory().to(dev, non_blocking=True)


def eval_epoch(model, config, opt, write_jsonl=True, rows_per_forward=ROWS_PER_FORWARD):
    """main/inference_qfvs.py eval_epoch on the device -> {'F', 'R', 'P'}; write_jsonl=False is main/train_qfvs.py's eval_epoch.

    Reads what the reference reads, from the same relative paths: data/qfvs/txt_clip/<txt_feature>.pkl, the processed
    P0<v>_<vid_feature>.h5 features (h5py), the oracle summaries of video v (os.walk order) and ./eval/Tags.mat (once), and writes
    the same ./plot/<dset_name>/<qfvs_split>.jsonl lines.  The forwards are batched: the query files are grouped by their two
    concept token counts and each group runs, per query variant, one forward of files x max_segment_num samples, at most
    rows_per_forward samples each (ROWS_PER_FORWARD by default).  Samples do not interact in the forward, so every row equals
    the reference's per-file forward bit for bit; the ensemble needs one forward per variant where the reference runs two, and
    without qfvs_score_gather only the both-concepts variant runs (the other two do not reach the score).  After each chunk one
    univtg_qfvs_eval_select launch forms the scores, the top k and the machine-side tag masks; one univtg_qfvs_match launch
    matches every file and one device-to-host copy brings back scores, top indices and matched weights.  p, r and f1 are
    calculate_semantic_matching's numpy expressions; no host synchronisation happens per chunk or per file.

    Refusals come after the JSONL file is opened, as the reference opens it first, and before any launch, so the file is left
    empty (the reference keeps the lines of the files before a failing one): ValueError for k = int(n * top_percent) == 0 (the reference's
    scikit-learn error), an empty ground-truth summary, more than 1,024 shots in a summary, tags that are not 0 / 1 or wider than
    64 columns, and more than 8,192 kept positions; IndexError for a ground-truth index outside the tag rows (negative indices
    wrap, as numpy's do) and a seg_len outside the mask grid; RuntimeError for features whose [S, Lf] differ from
    [max_segment_num, max_frame_num] (the reference's masked_select error) and for a model that is not on a CUDA device."""
    import pickle

    import h5py

    model.eval()
    f1_sum = 0
    p_sum = 0
    r_sum = 0
    assert len(config["test_videos"]) == 1
    video_id = config["test_videos"][0]
    with open(f"./data/qfvs/txt_clip/{config['txt_feature']}.pkl", "rb") as f:
        embedding = pickle.load(f)
    feat = h5py.File(f"./data/qfvs/processed/P0{video_id}_{config['vid_feature']}.h5", "r")
    features = torch.from_numpy(feat["features"][()])
    seg_len = [int(x) for x in np.asarray(feat["seg_len"][()]).reshape(-1)]
    summary_dir = SUMMARY_DIR + str(video_id)
    S, Lf = config["max_segment_num"], config["max_frame_num"]
    f_write = open(os.path.join("./plot", opt.dset_name, str(opt.qfvs_split) + ".jsonl"), "w") if write_jsonl else None
    try:
        entries = [files for _, _, files in os.walk(summary_dir)]
        for files in entries:
            evaluation_num = len(files)
        files = [x for fs in entries for x in fs]
        queries = _read_queries(summary_dir, files, embedding)
        mask = np.zeros((S, Lf), dtype=bool)
        for j in range(len(seg_len)):
            if seg_len[j] > 0 and (j >= S or seg_len[j] > Lf):
                raise IndexError(f"mask_GT: segment {j} of {seg_len[j]} frames is outside the {S} x {Lf} grid")
            mask[j, :max(seg_len[j], 0)] = True
        if queries:
            host = _epoch_host(model, config, opt, load_videos_tag(mat_path="./eval/Tags.mat")[video_id - 1], features, mask,
                               queries, rows_per_forward)
            res = _run_epoch(model, host, queries, features, mask)
            for q, qu in enumerate(queries):
                s = np.float64(res["s"][q])
                p, r, f1 = precision_recall_f1(s, host["k"], len(qu["gt"]))
                if f_write is not None:
                    entry = {"concept1": qu["c1"], "concept2": qu["c2"], "score": res["score"][q].tolist(),
                             "top_percent": config["top_percent"], "top_pred": res["top"][q].tolist(), "gt": qu["gt"],
                             "p": p, "r": r, "f1": f1, "shots": host["shots"]}
                    f_write.write(json.dumps(entry) + "\n")
                f1_sum += f1
                r_sum += r
                p_sum += p
    finally:
        if f_write is not None:
            f_write.close()
    return {"F": round(100 * f1_sum / evaluation_num, 2),
            "R": round(100 * r_sum / evaluation_num, 2),
            "P": round(100 * p_sum / evaluation_num, 2)}


def _read_queries(summary_dir, files, embedding):
    out = []
    for file in files:
        with open(summary_dir + "/" + file, "r") as f:
            gt = [int(line.strip()) for line in f.readlines()]
        c1, c2 = file.split("_")[0:2]
        c1, c2 = TRANSFER.get(c1, c1), TRANSFER.get(c2, c2)
        t1, t2 = (torch.from_numpy(l2_normalize_np_array(embedding[c])).to(torch.float32) for c in (c1, c2))
        if t1.dim() != 2 or t2.dim() != 2:
            raise ValueError(f"{file}: concept embeddings must be [tokens, dim], got {list(t1.shape)} and {list(t2.shape)}")
        out.append({"file": file, "c1": c1, "c2": c2, "gt": [x - 1 for x in gt], "t1": t1, "t2": t2})
    return out


def _epoch_host(model, config, opt, tags, features, mask, queries, rows_per_forward):
    """Everything the epoch needs from the host, checked before any launch: sizes, the select positions and tag table, and the
    matching's ground-truth side."""
    mode = output_type(opt, config)
    S, Lf = mask.shape
    if features.dim() != 3 or tuple(features.shape[:2]) != (S, Lf):
        raise RuntimeError(f"the model outputs [S, Lf] = {list(features.shape[:2])} do not match mask_GT {[S, Lf]}")
    tags = np.asarray(tags)
    shots = tags.shape[0]
    pos = np.flatnonzero(mask.reshape(-1))
    n = min(len(pos), shots)
    k = int(n * config["top_percent"])
    if k == 0:
        raise ValueError("Found array with 0 sample(s) (shape=(0, %d)) while a minimum of 1 is required: empty machine summary"
                         % (tags.shape[1] if tags.ndim == 2 else 0))
    if n > SELECT_MAX_N:
        raise ValueError(f"QFVS eval_epoch: {n} kept positions per query, at most {SELECT_MAX_N}")
    if k > MAX_SIDE:
        raise ValueError(f"semantic matching: each summary must hold 1..{MAX_SIDE} shots (k = {k})")
    table = tag_masks(tags)
    gts = []
    for qu in queries:
        rows = tags[qu["gt"]]
        _check_not_empty(rows, "ground-truth")
        if rows.shape[0] > MAX_SIDE:
            raise ValueError(f"semantic matching: each summary must hold 1..{MAX_SIDE} shots ({qu['file']}: {rows.shape[0]})")
        gts.append(table[np.asarray(qu["gt"], dtype=np.int64) % shots])
    # chunks: the files sharing both concept token counts, at most rows_per_forward // S files each; the pools hold the queries
    # in chunk order (slot[q] = pool row of file q), and the matching's ground-truth side is packed in that order too
    groups = {}
    for q, qu in enumerate(queries):
        groups.setdefault((qu["t1"].shape[0], qu["t2"].shape[0]), []).append(q)
    per = max(1, rows_per_forward // S)
    chunks = [(key, m[c:c + per]) for key, m in groups.items() for c in range(0, len(m), per)]
    order = [q for _, chunk in chunks for q in chunk]
    slot = np.empty(len(queries), dtype=np.int64)
    slot[order] = np.arange(len(queries))
    if _model_device(model).type != "cuda":
        raise RuntimeError("univtg_b200: the QFVS eval_epoch runs on CUDA only (no CPU path); move the model to a CUDA device")
    Q = len(queries)
    b_off = np.concatenate([[0], np.cumsum([len(gts[q]) for q in order])]).astype(np.int32)
    return {"mode": mode, "gather": int(config["qfvs_score_gather"] > 0), "shots": shots, "n": n, "k": k,
            "max_side": int(max(k, max(len(b) for b in gts))), "chunks": chunks, "slot": slot,
            "parts": [np.concatenate([gts[q] for q in order]).astype(np.uint64), table.astype(np.uint64), b_off,
                      (np.arange(Q + 1) * k).astype(np.int32), pos[:n].astype(np.int32)]}


def _run_epoch(model, host, queries, features, mask):
    """The device part: batched forwards, one select per chunk, one matching, one read-back."""
    lib = _lib.load_library()
    dev = _model_device(model)
    S, Lf = mask.shape
    Q, n, k, mode, gather = len(queries), host["n"], host["k"], host["mode"], host["gather"]
    with torch.no_grad(), torch.cuda.device(dev):
        # one upload of the host side: b, tag table, b_off, a_off, pos, then every query's texts
        parts = host["parts"]
        raw = [x.view(np.uint8) for x in parts]
        offs = np.concatenate([[0], np.cumsum([len(r) for r in raw])])
        texts = [torch.cat([qu["t1"], qu["t2"]]).numpy() for qu in queries]
        t_offs = offs[-1] + np.concatenate([[0], np.cumsum([t.nbytes for t in texts])])
        buf = _pinned(np.concatenate(raw + [t.reshape(-1).view(np.uint8) for t in texts]), dev)
        base = buf.data_ptr()
        at = lambda i: _lib.c_void_p(base + int(offs[i]))  # noqa: E731
        Dt = texts[0].shape[1]

        def text(q, lo, hi):
            L = queries[q]["t1"].shape[0] + queries[q]["t2"].shape[0]
            return buf[int(t_offs[q]):int(t_offs[q + 1])].view(torch.float32).view(L, Dt)[lo:hi]

        tef_st = torch.arange(0, Lf, 1.0) / Lf
        tef = torch.stack([tef_st, tef_st + 1.0 / Lf], dim=1).repeat(S, 1, 1)
        video = torch.cat([features.to(torch.float32), tef], dim=-1).pin_memory().to(dev, non_blocking=True)
        vmask = torch.from_numpy(mask.astype(np.float32)).pin_memory().to(dev, non_blocking=True)

        score = torch.empty(Q, n, dtype=torch.float32, device=dev)
        top = torch.empty(Q, k, dtype=torch.int32, device=dev)
        a = torch.empty(Q, k, dtype=torch.int64, device=dev)
        s = torch.empty(Q, dtype=torch.float64, device=dev)
        q0 = 0
        for (L1, L2), chunk in host["chunks"]:  # pool slots q0 .. q0 + F - 1 in chunk order
            F = len(chunk)
            vid = video.repeat(F, 1, 1)
            vm = vmask.repeat(F, 1)
            outs = [None, None, None]
            for v, (lo, hi) in enumerate(((0, L1), (L1, L1 + L2), (0, L1 + L2))):
                if v < 2 and not gather:
                    continue
                txt = torch.stack([text(q, lo, hi) for q in chunk]).repeat_interleave(S, dim=0)
                o = model(src_vid=vid, src_vid_mask=vm, src_txt=txt, src_txt_mask=torch.ones(F * S, hi - lo, device=dev))
                outs[v] = [o[key].detach().to(torch.float32).contiguous() for key in ("pred_logits", "saliency_scores")]
            ptrs = [_lib.ptr(o[i]) if o is not None else None for o in outs for i in (0, 1)]
            _lib.check(lib.univtg_qfvs_eval_select(*ptrs, at(4), at(1), F, S * Lf, n, k, mode, gather, q0, _lib.ptr(score),
                                                   _lib.ptr(top), _lib.ptr(a), _lib.stream_ptr()), "univtg_qfvs_eval_select")
            q0 += F
        _lib.check(lib.univtg_qfvs_match(_lib.ptr(a), at(3), at(0), at(2), Q, host["max_side"], _lib.ptr(s), _lib.stream_ptr()),
                   "univtg_qfvs_match")
        arena = torch.cat([t.view(torch.uint8).reshape(-1) for t in (s, score, top)]).cpu().numpy()
    slot = host["slot"]
    out, o = {}, 0
    for name, cnt, dt in (("s", Q, np.float64), ("score", Q * n, np.float32), ("top", Q * k, np.int32)):
        nb = cnt * np.dtype(dt).itemsize
        out[name] = arena[o:o + nb].view(dt).reshape(Q, -1)[slot]  # file order
        o += nb
    out["s"] = out["s"][:, 0]
    return out

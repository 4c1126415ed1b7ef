"""CLIP-teacher pseudo labels on the GPU: the reference's teacher/clip2label.py.

UniVTG's pre-training labels come from CLIP: each video's clip features are compared with the text features of ~20k
OpenImages class prompts ("a photo of a {x}", teacher/label2feature.py), the 5 classes with the largest summed cosine become
queries, and each query's curve cos // 0.05 gives its saliency scores and the windows of its maximum.  This module computes
the same labels through the CUDA library (include/univtg_b200.h, univtg_teacher_*):

    labeler = PseudoLabeler(torch.from_numpy(np.load("class_text.npz")["pooler_output"]).cuda(), "oidv6-class-descriptions.csv")
    samples = labeler([feats_a, feats_b], ["vid_a", "vid_b"])    # the reference's dicts
    write_pseudo_labels("curve_5_window.jsonl", "data/videocc/vid_clip", labeler, slowfast_dir="data/videocc/vid_slowfast")

The ranking key is the float64 sum over clips of the float64 cosines (ties to the lower class index) and each curve value is
the float64 cosine rounded to float32, then Python's `//`; the lines equal those of oracle/teacher_oracle.py byte for byte.
Videos come out in the order given (write_pseudo_labels sorts them by name) and a video's lines in rank order.  CUDA only.
"""
import csv
import json
import math
import os

import numpy as np
import torch

from . import _lib

MAX_TOPK = 16
MAX_DIM = 1024
MAX_CLIPS = 65535           # clips per video
MIN_TH = 2.0 ** -30         # curve bins (|cos| / th + 1) stay inside int32
APPROX_BYTES = 1 << 27      # a chunk's approximate score matrix [videos, C rounded up to 16] f32 stays within 128 MiB
FEATURE_BYTES = 1 << 30     # and its packed clip features within 1 GiB (or one video)
_NEG_ZERO = np.iinfo(np.int32).min


def read_class_names(path):
    """The class names clip2label.py indexes: its JSON list, or the DisplayName column of oidv6-class-descriptions.csv with the
    header skipped (teacher/csv2json.py)."""
    if path.endswith(".csv"):
        with open(path, newline="", encoding="utf-8") as f:
            rows = list(csv.reader(f, delimiter=","))
        return [r[1] for r in rows[1:]]
    with open(path, encoding="utf-8") as f:
        names = json.load(f)
    if not isinstance(names, list):
        raise ValueError(f"{path}: expected a JSON list of class names")
    return names


class _BinText(dict):
    """'[19.0]'-style text of a curve bin (json.dumps of [float(bin)]), made once per value."""

    def __missing__(self, b):
        t = "[-0.0]" if b == _NEG_ZERO else "[" + repr(float(b)) + "]"
        self[b] = t
        return t


class PseudoLabeler:
    """clip2label.py's labelling with a fixed class table.

    class_features: float32 [C, D] CUDA tensor (class_text.npz['pooler_output']), D <= 1024.
    names: the C class names, or a path to the reference's JSON list or to oidv6-class-descriptions.csv.
    topk (1..16), th (the curve bin width) and clip_len (seconds per clip) are clip2label.py's constants."""

    def __init__(self, class_features, names, topk=5, th=0.05, clip_len=2):
        if not torch.is_tensor(class_features) or class_features.device.type != "cuda":
            raise RuntimeError("PseudoLabeler: class_features must be a CUDA tensor (univtg_b200 has no CPU path)")
        if class_features.dtype != torch.float32 or class_features.dim() != 2:
            raise ValueError(f"PseudoLabeler: class_features must be float32 [C, D], got {class_features.dtype} "
                             f"{tuple(class_features.shape)}")
        C, D = class_features.shape
        if C < 1 or not 1 <= D <= MAX_DIM:
            raise ValueError(f"PseudoLabeler: need C >= 1 and D in 1..{MAX_DIM}, got [{C}, {D}]")
        if isinstance(names, (str, os.PathLike)):
            names = read_class_names(os.fspath(names))
        names = list(names)
        if len(names) != C:
            raise ValueError(f"PseudoLabeler: {len(names)} names for {C} class rows")
        if isinstance(topk, bool) or not isinstance(topk, int) or not 1 <= topk <= MAX_TOPK:
            raise ValueError(f"PseudoLabeler: topk must be an int in 1..{MAX_TOPK}, got {topk!r}")
        th = float(th)
        if not (math.isfinite(th) and th >= MIN_TH):
            raise ValueError(f"PseudoLabeler: th must be finite and >= 2^-30, got {th!r}")
        if isinstance(clip_len, bool) or not isinstance(clip_len, (int, float)) or not clip_len > 0:
            raise ValueError(f"PseudoLabeler: clip_len must be a positive number, got {clip_len!r}")
        self.C, self.D, self.topk, self.th, self.clip_len = C, D, topk, th, clip_len
        self.names = names
        self.fallback_videos = 0  # videos of the last call rescored over every class
        self._lib = _lib.load_library()
        self._dev = class_features.device
        self._cls = class_features.contiguous()
        self._cls_ws = torch.empty(self._lib.univtg_teacher_class_bytes(C, D), dtype=torch.uint8, device=self._dev)
        with torch.cuda.device(self._dev):
            _lib.check(self._lib.univtg_teacher_prepare_classes(_lib.ptr(self._cls), C, D, _lib.ptr(self._cls_ws), _lib.stream_ptr()),
                       "univtg_teacher_prepare_classes")
        self._query = [json.dumps(n) for n in names]
        self._ids = {}
        self._bins = _BinText()
        c16 = (C + 15) // 16 * 16
        self._max_videos = max(1, APPROX_BYTES // (4 * c16))
        self._max_clips = max(MAX_CLIPS, FEATURE_BYTES // (4 * D))

    # ---- device ----
    def _check(self, features, vids):
        if isinstance(vids, str) or len(features) != len(vids):
            raise ValueError(f"PseudoLabeler: {len(features)} feature arrays for {len(vids)} video names")
        lens = []
        for i, f in enumerate(features):
            if torch.is_tensor(f):
                if f.device.type != "cuda":
                    raise RuntimeError("PseudoLabeler: feature tensors must be on CUDA (univtg_b200 has no CPU path)")
                dt = f.dtype == torch.float32
            elif isinstance(f, np.ndarray):
                dt = f.dtype == np.float32
            else:
                raise ValueError(f"PseudoLabeler: features[{i}] is a {type(f).__name__}, not a numpy array or tensor")
            T = f.shape[0] if f.ndim >= 1 else -1
            if T != 0 and (not dt or f.ndim != 2 or f.shape[1] != self.D):
                raise ValueError(f"PseudoLabeler: features[{i}] must be float32 [T, {self.D}], got {f.dtype} {tuple(f.shape)}")
            if T > MAX_CLIPS:
                raise ValueError(f"PseudoLabeler: features[{i}] has {T} clips (at most {MAX_CLIPS})")
            lens.append(T)
        return lens

    def _chunks(self, lens):
        cur, clips = [], 0
        for i, T in enumerate(lens):
            if T == 0:  # clip2label.py:64-65
                continue
            if cur and (len(cur) == self._max_videos or clips + T > self._max_clips):
                yield cur
                cur, clips = [], 0
            cur.append(i)
            clips += T
        if cur:
            yield cur

    def _label_chunk(self, features, lens, chunk):
        """One H2D copy of the packed features and offsets, the library call, one D2H copy of the results."""
        V, K, D = len(chunk), self.topk, self.D
        off = np.zeros(V + 1, dtype=np.int32)
        np.cumsum([lens[i] for i in chunk], out=off[1:])
        S = int(off[-1])
        if any(torch.is_tensor(features[i]) for i in chunk):
            feats = torch.cat([torch.as_tensor(features[i]).to(self._dev).reshape(-1) for i in chunk] +
                              [torch.from_numpy(off.view(np.float32)).to(self._dev)])
        else:
            host = torch.empty(S * D + V + 1, dtype=torch.float32, pin_memory=True)
            hn = host.numpy()
            for i, lo, hi in zip(chunk, off[:-1], off[1:]):
                hn[lo * D:hi * D] = features[i].reshape(-1)
            hn[S * D:].view(np.int32)[:] = off
            feats = host.to(self._dev, non_blocking=True)
        offsets = feats[S * D:]
        ws = torch.empty(self._lib.univtg_teacher_chunk_bytes(V, S, self.C, D), dtype=torch.uint8, device=self._dev)
        out = torch.empty(2 * V * K + 2 * S * K + 1, dtype=torch.int32, device=self._dev)
        with torch.cuda.device(self._dev):
            _lib.check(self._lib.univtg_teacher_label(_lib.ptr(self._cls), _lib.ptr(self._cls_ws), self.C, D, _lib.ptr(feats),
                                                      _lib.ptr(offsets), V, S, K, self.th, _lib.ptr(ws), ws.numel(), _lib.ptr(out),
                                                      _lib.stream_ptr()), "univtg_teacher_label")
        res = out.cpu().numpy()
        idx = res[:V * K].reshape(V, K)
        nwin = res[V * K:2 * V * K].reshape(V, K)
        win = res[2 * V * K:2 * V * K + S * K].view(np.uint32).reshape(S, K)
        bins = res[2 * V * K + S * K:-1].reshape(S, K)
        self.fallback_videos += int(res[-1])
        return off, idx, nwin, win, bins

    def _rows(self, features, vids):
        """(vid, T, class, windows, bin column) of every line, videos in the given order, ranks in order."""
        lens = self._check(features, vids)
        self.fallback_videos = 0
        cl = self.clip_len
        for chunk in self._chunks(lens):
            off, idx, nwin, win, bins = self._label_chunk(features, lens, chunk)
            for v, i in enumerate(chunk):
                lo, hi = int(off[v]), int(off[v + 1])
                for r in range(self.topk):
                    n = int(nwin[v, r])
                    if idx[v, r] < 0 or n == 0:
                        continue
                    w = win[lo:lo + n, r].tolist()
                    yield vids[i], hi - lo, int(idx[v, r]), [[(x >> 16) * cl, ((x & 0xffff) + 1) * cl] for x in w], bins[lo:hi, r]

    # ---- public ----
    def __call__(self, features, vids):
        """The reference's sample dicts (one per line of curve_{topk}_window.jsonl) of the given videos.  features: float32
        [T_i, D] numpy arrays or CUDA tensors; videos with T = 0 are skipped."""
        out = []
        for vid, T, c, windows, b in self._rows(features, vids):
            out.append({"qid": c, "query": self.names[c], "duration": float(T * self.clip_len), "vid": vid,
                        "relevant_clip_ids": list(range(T)), "relevant_windows": windows,
                        "saliency_scores": [[-0.0] if x == _NEG_ZERO else [float(x)] for x in b.tolist()]})
        return out

    def lines(self, features, vids):
        """json.dumps of each sample of __call__, built from cached pieces."""
        out = []
        bt = self._bins
        for vid, T, c, windows, b in self._rows(features, vids):
            ids = self._ids.get(T)
            if ids is None:
                ids = self._ids[T] = json.dumps(list(range(T)))
            out.append('{"qid": %d, "query": %s, "duration": %r, "vid": %s, "relevant_clip_ids": %s, "relevant_windows": %s, '
                       '"saliency_scores": [%s]}' % (c, self._query[c], float(T * self.clip_len), json.dumps(vid), ids,
                                                     json.dumps(windows), ", ".join([bt[x] for x in b.tolist()])))
        return out


def write_pseudo_labels(out_path, clip_dir, labeler, slowfast_dir=None, batch_videos=4096):
    """clip2label.py's __main__: label every {vid}.npz of clip_dir (its 'features' array), restricted to the names also in
    slowfast_dir when that is given, and write the lines to out_path, videos sorted by name.  Returns the number of lines."""
    if batch_videos < 1:
        raise ValueError("write_pseudo_labels: batch_videos must be >= 1")
    names = set(os.listdir(clip_dir))
    if slowfast_dir is not None:
        names &= set(os.listdir(slowfast_dir))
    names = sorted(n for n in names if n.endswith(".npz"))
    n_lines = 0
    with open(out_path, "w") as f:
        for s in range(0, len(names), batch_videos):
            batch = names[s:s + batch_videos]
            feats = []
            for n in batch:
                with np.load(os.path.join(clip_dir, n)) as z:
                    feats.append(z["features"])
            lines = labeler.lines(feats, [n[:-4] for n in batch])
            for line in lines:
                f.write(line)
                f.write("\n")
            n_lines += len(lines)
    return n_lines

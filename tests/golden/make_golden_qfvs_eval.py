#!/usr/bin/env python
"""Writes tests/golden/reference_qfvs_eval.json: what the live reference's QFVS evaluation epochs (main/inference_qfvs.py and
main/train_qfvs.py eval_epoch) write and return on the seeded cases below, so the restatement (tests/qfvs_eval_oracle.py) and
the device epoch (univtg_b200.qfvs.eval_epoch) stay pinned without the reference.

Each case builds its inputs with univtg_b200.synth.write_qfvs_eval_tree in a temporary directory (the pickle, the features, the
oracle summaries and a savemat-written Tags.mat with the released file's layout), changes into it and runs both unmodified
eval_epoch functions on the CPU: h5py is univtg_b200.synth.h5py_stub(), `.cuda()` and `.to('cuda')` stay on the CPU, and the
model is univtg_b200.synth.QFVSReplayModel.  Stored per case: its parameters, the JSONL lines by file name, both returned dicts
(json.dumps strings) or the exception type both raise, and the JSONL text when an exception left it.  A case whose scores tie
exactly among the top k + 1 of some file is drawn again with the next seed (torch.topk's order among ties is not what the
golden pins).

Usage: python tests/golden/make_golden_qfvs_eval.py <path to a showlab/UniVTG checkout>"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from univtg_b200 import synth  # noqa: E402

FILES3 = (("Beach", "Car"), ("Cupglass", "Tree"), ("Musicalinstrument", "Petsanimal"))
FILES6 = FILES3 + (("Sky", "Food"), ("Water", "Book"), ("Car", "Sky"))
BASE = dict(seed=1, video_id=1, S=4, Lf=16, seg_len=(16, 16, 16, 5), shots=(60, 60, 60, 60), files=FILES3, gt_sizes=(5, 3, 8),
            gt_extra=(), tokens=None, top_percent=0.1, ensemble=1, gather=1, f_coef=10.0, s_coef=0.1)
CASES = [
    dict(name="ensemble_gather"),
    dict(name="ensemble_no_gather", seed=2, gather=0, files=FILES6),
    dict(name="logits_no_ensemble", seed=3, ensemble=0, top_percent=0.5),
    dict(name="logits_s_intra_0", seed=4, s_coef=0.0, gather=0, top_percent=0.3),
    dict(name="saliency_f_0", seed=5, f_coef=0.0, files=FILES6),
    dict(name="k1", seed=6, top_percent=0.02),
    dict(name="feats_beyond_tags", seed=7, video_id=2, shots=(60, 40, 60, 60), top_percent=0.25),
    dict(name="video4_ragged", seed=8, video_id=4, S=5, Lf=12, seg_len=(12, 12, 3), shots=(60, 60, 60, 30), files=FILES6),
    dict(name="one_token_each", seed=9, tokens={c: 1 for c in synth.QFVS_CONCEPTS + ("Glass", "Instrument", "Animal")}),
    dict(name="gt_negative_wraps", seed=10, gt_extra=((0,), (), ())),
    dict(name="k0", seed=11, top_percent=0.001),
]


def case_params(c):
    p = dict(BASE)
    p.update(c)
    return p


def build_tree(p, root):
    synth.write_qfvs_eval_tree(root, p["seed"], video_id=p["video_id"], S=p["S"], Lf=p["Lf"], seg_len=p["seg_len"], shots=p["shots"],
                               files=p["files"], tokens=p["tokens"], gt_sizes=p["gt_sizes"], gt_extra=p["gt_extra"])


def case_config(p):
    return synth.qfvs_eval_config(test_videos=[p["video_id"]], max_segment_num=p["S"], max_frame_num=p["Lf"],
                                  top_percent=p["top_percent"], qfvs_score_ensemble=p["ensemble"], qfvs_score_gather=p["gather"])


def case_opt(p):
    return synth.qfvs_eval_opt(qfvs_split=p["video_id"], f_loss_coef=p["f_coef"], s_loss_intra_coef=p["s_coef"])


def jsonl_path(p):
    return os.path.join("plot", "qfvs", f"{p['video_id']}.jsonl")


def lines_by_file(p, text):
    """JSONL text -> {oracle summary file name: line} (the reference writes one line per file, in os.walk order)."""
    names = {"{}_{}".format(*synth_transfer(c)): "{}_{}_oracle.txt".format(*c) for c in p["files"]}
    out = {}
    for line in text.splitlines():
        e = json.loads(line)
        out[names["{}_{}".format(e["concept1"], e["concept2"])]] = line
    return out


def synth_transfer(c):
    t = {"Cupglass": "Glass", "Musicalinstrument": "Instrument", "Petsanimal": "Animal"}
    return tuple(t.get(x, x) for x in c)


def has_tie(line, k):
    s = sorted(json.loads(line)["score"], reverse=True)[:k + 1]
    return any(a == b for a, b in zip(s, s[1:]))


def run(fn, model, p, root, *args):
    """Run one eval_epoch in root -> (result json or None, exception type name or None, JSONL text or None)."""
    cwd = os.getcwd()
    os.chdir(root)
    try:
        res, err = json.dumps(fn(model, case_config(p), case_opt(p), *args)), None
    except Exception as e:  # noqa: BLE001 - the golden records which exception the reference raises
        res, err = None, type(e).__name__
    finally:
        os.chdir(cwd)
    path = os.path.join(root, jsonl_path(p))
    text = open(path).read() if os.path.exists(path) else None
    if text is not None:
        os.remove(path)
    return res, err, text


def main():
    sys.path.insert(0, os.path.abspath(sys.argv[1]))
    from make_golden_eval_epoch import stub_reference_deps

    sys.modules["h5py"] = synth.h5py_stub()
    stub_reference_deps()  # nncore
    import torch

    torch.Tensor.cuda = lambda self, *a, **k: self  # every tensor stays on the CPU
    to = torch.Tensor.to
    torch.Tensor.to = lambda self, *a, **k: to(self, *("cpu" if x == "cuda" else x for x in a), **k)
    import main.inference_qfvs as I
    import main.train_qfvs as T

    cases = []
    for c in CASES:
        p = case_params(c)
        for _ in range(20):
            with tempfile.TemporaryDirectory() as tmp:
                build_tree(p, tmp)
                res_i, err_i, text = run(I.eval_epoch, synth.QFVSReplayModel(p["seed"]), p, tmp)
                res_t, err_t, _ = run(T.eval_epoch, synth.QFVSReplayModel(p["seed"]), p, tmp)
            lines = lines_by_file(p, text) if err_i is None else {}
            k = len(json.loads(next(iter(lines.values())))["top_pred"]) if lines else 0
            if not any(has_tie(x, k) for x in lines.values()):
                break
            p["seed"] += 1000
        else:
            raise RuntimeError(f"{p['name']}: no tie-free draw")
        cases.append({"params": p, "lines": lines, "inference": res_i, "train": res_t, "error": err_i, "train_error": err_t,
                      "jsonl_on_error": text if err_i else None})
        print(p["name"], "seed", p["seed"], "files", len(lines), "->", res_i or err_i, "/", res_t or err_t)
    out = {"torch": torch.__version__, "cases": cases}
    path = os.path.join(HERE, "reference_qfvs_eval.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", path, len(cases), "cases")


if __name__ == "__main__":
    main()

"""Time the QFVS evaluation epoch (main/inference_qfvs.py eval_epoch) on one GPU, in one call.

    python tools/qfvs_eval_cost.py [--files 45] [--epochs 5] [--warmup 1] [--json out.json]

One test video at the real sizes: S = 20 segments of Lf = 200 frames, the last one ragged (137 frames, 3,937 kept positions),
the four Tags.mat shot counts 2,783 / 3,692 / 2,152 / 3,588 (videos 1-4) with top_percent 0.02, which gives machine summaries of
55 / 73 / 43 / 71 shots (the summary sizes of DESIGN §5.7) and ground-truth summaries of the same sizes; cfg2 model dims with
Dv = 2818 and 8 tokens per concept, as tools/qfvs_cost.py assumes.  --files query files per video (45 by default).  Two
output configurations: the reference's defaults (qfvs_score_ensemble = qfvs_score_gather = -1: pred_logits of the
both-concepts query) and the ensemble with gathering (1 / 1).  The inputs are written to a temporary directory (features
through univtg_b200.synth.h5py_stub).

Arms, alternated epoch by epoch after a warm-up of each: (a) univtg_b200.qfvs.eval_epoch; (b) the reference's per-file
arrangement restated here with the same model (three forwards per file, six with the ensemble, masked_select, the sums, topk,
Tags.mat loaded per file, qfvs.calculate_semantic_matching on the device per file).  The tool checks that both arms write
the same JSONL lines, and reports per configuration and video the median and min-max wall time of an epoch (host clock
around the whole call, which ends with a device-to-host copy), with the GPU's name and power limit read in the same call.
"""
import argparse
import contextlib
import json
import os
import pickle
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from clip_cost import gpu_info  # noqa: E402
from univtg_b200 import qfvs, synth  # noqa: E402
from univtg_b200.qfvs import build_model  # noqa: E402

S, LF, SEG_LEN, TOKENS = 20, 200, (200,) * 19 + (137,), 8
SHOTS = (2783, 3692, 2152, 3588)
SUMMARY = (55, 73, 43, 71)


def per_file_epoch(model, config, opt):
    """The reference's loop body, file by file, on this library's model and device matching."""
    model.eval()
    f1_sum = p_sum = r_sum = 0
    video_id = config["test_videos"][0]
    with open(f"./data/qfvs/txt_clip/{config['txt_feature']}.pkl", "rb") as f:
        embedding = pickle.load(f)
    feat = sys.modules["h5py"].File(f"./data/qfvs/processed/P0{video_id}_{config['vid_feature']}.h5", "r")
    features = torch.from_numpy(feat["features"][()])
    seg_len = torch.from_numpy(feat["seg_len"][()])
    mode = qfvs.output_type(opt, config)
    keys = {0: ["pred_logits"], 1: ["saliency_scores"], 2: ["pred_logits", "saliency_scores"]}[mode]
    with open(os.path.join("./plot", opt.dset_name, str(opt.qfvs_split) + ".jsonl"), "w") as f_write:
        d = qfvs.SUMMARY_DIR + str(video_id)
        for _, _, files in os.walk(d):
            n_files = len(files)
            mask = torch.zeros(config["max_segment_num"], config["max_frame_num"], dtype=torch.bool).cuda()
            for j in range(len(seg_len)):
                for k in range(seg_len[j]):
                    mask[j][k] = 1
            for file in files:
                with open(d + "/" + file) as f:
                    gt = [int(x.strip()) - 1 for x in f.readlines()]
                c1, c2 = (qfvs.TRANSFER.get(c, c) for c in file.split("_")[0:2])
                t1, t2 = (torch.from_numpy(qfvs.l2_normalize_np_array(embedding[c])).float() for c in (c1, c2))
                seq = features.float().cuda()
                tef_st = torch.arange(0, LF, 1.0) / LF
                seq = torch.cat([seq, torch.stack([tef_st, tef_st + 1.0 / LF], 1).cuda().repeat(S, 1, 1)], -1)
                vm = mask.float()
                inputs = [dict(src_vid=seq, src_vid_mask=vm, src_txt=t.cuda().repeat(S, 1, 1), src_txt_mask=torch.ones(S, t.shape[0]).cuda())
                          for t in (t1, t2, torch.cat([t1, t2]))]
                tags = qfvs.load_videos_tag(mat_path="./eval/Tags.mat")
                with torch.no_grad():
                    if mode == 2:
                        sc = [torch.zeros(int(mask.sum().item())).cuda() for _ in range(3)]
                        for key in keys:
                            for i in range(3):
                                sc[i] += model(**inputs[i])[key].squeeze().masked_select(mask)
                    else:
                        sc = [model(**inp)[keys[0]].squeeze().masked_select(mask) for inp in inputs]
                    score = sc[2] + sc[0] + sc[1] if config["qfvs_score_gather"] > 0 else sc[2]
                    score = score[:min(score.shape[0], tags[video_id - 1].shape[0])]
                    _, top = score.topk(int(score.shape[0] * config["top_percent"]))
                    p, r, f1 = qfvs.calculate_semantic_matching(list(top.cpu().numpy()), gt, tags, video_id=video_id - 1)
                    entry = {"concept1": c1, "concept2": c2, "score": score.tolist(), "top_percent": config["top_percent"],
                             "top_pred": top.tolist(), "gt": gt, "p": p, "r": r, "f1": f1, "shots": tags[video_id - 1].shape[0]}
                    f_write.write(json.dumps(entry) + "\n")
                    f1_sum += f1
                    r_sum += r
                    p_sum += p
    return {"F": round(100 * f1_sum / n_files, 2), "R": round(100 * r_sum / n_files, 2), "P": round(100 * p_sum / n_files, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=45)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--videos", default="1,2,3,4")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "qfvs_eval_cost.py measures on a GPU; there is no CPU measurement"
    torch.backends.cuda.matmul.allow_tf32 = False
    sys.modules["h5py"] = synth.h5py_stub()
    cfg = synth.CONFIGS["cfg2"]
    model, _ = build_model(synth.reference_args(cfg, device="cuda", dset_type="vs"))
    model.load_state_dict(synth.make_state_dict(cfg, seed=4), strict=True)
    model.cuda().eval()
    names = synth.QFVS_CONCEPTS
    pairs = [(a, b) for a in names for b in names if a != b][:args.files]
    rows = []
    with tempfile.TemporaryDirectory() as tmp, contextlib.chdir(tmp):
        for v in (int(x) for x in args.videos.split(",")):
            synth.write_qfvs_eval_tree(tmp, 40 + v, video_id=v, S=S, Lf=LF, seg_len=SEG_LEN, dv=cfg["v_feat_dim"] - 2, dt=cfg["t_feat_dim"],
                                       shots=SHOTS, files=pairs, tokens={c: TOKENS for c in names + ("Glass", "Instrument", "Animal")},
                                       gt_sizes=(SUMMARY[v - 1],))
            for label, ens in (("default", -1), ("ensemble_gather", 1)):
                config = synth.qfvs_eval_config(test_videos=[v], top_percent=0.02, qfvs_score_ensemble=ens, qfvs_score_gather=ens)
                opt = synth.qfvs_eval_opt(qfvs_split=v)
                arms = {"eval_epoch": lambda: qfvs.eval_epoch(model, config, opt),
                        "per_file": lambda: per_file_epoch(model, config, opt)}
                text, res = {}, {}
                for name, fn in arms.items():
                    for _ in range(args.warmup):
                        res[name] = fn()
                    with open(os.path.join("plot", "qfvs", f"{v}.jsonl")) as f:
                        text[name] = f.read()
                ms = {name: [] for name in arms}
                for _ in range(args.epochs):
                    for name, fn in arms.items():
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        fn()
                        torch.cuda.synchronize()
                        ms[name].append(1e3 * (time.perf_counter() - t0))
                same = sorted(text["eval_epoch"].splitlines()) == sorted(text["per_file"].splitlines())
                row = {"video": v, "shots": SHOTS[v - 1], "k": SUMMARY[v - 1], "config": label, "files": len(pairs),
                       "same_lines": same, "result": res,
                       "epoch_ms_median": {k: statistics.median(x) for k, x in ms.items()},
                       "epoch_ms_min_max": {k: [min(x), max(x)] for k, x in ms.items()}}
                row["speedup"] = row["epoch_ms_median"]["per_file"] / row["epoch_ms_median"]["eval_epoch"]
                print(json.dumps(row), flush=True)
                rows.append(row)
    result = {"gpu": gpu_info(), "shape": {"S": S, "Lf": LF, "seg_len_last": SEG_LEN[-1], "tokens_per_concept": TOKENS, "config": "cfg2"},
              "files": len(pairs), "epochs": args.epochs, "warmup": args.warmup, "rows_per_forward": qfvs.ROWS_PER_FORWARD, "rows": rows}
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)
    assert all(r["same_lines"] for r in rows), "the two arms wrote different lines"


if __name__ == "__main__":
    main()

"""Generate tests/golden/reference_clip.npz from an unmodified UniVTG checkout (CPU, fp32).

    python tests/golden/make_golden_clip.py <UniVTG checkout>

run_on_video/clip/model.py and run_on_video/preprocessing.py are loaded by file path (the package __init__ imports the
tokenizer, which needs ftfy).  For each small CLIP config of univtg_b200.synth the script regenerates the seeded state dict,
frames and token rows, asks the reference's build_model(state_dict) which architecture it infers, and evaluates the reference
CLIP in fp32 (build_model converts to fp16; the fp32 weights are loaded back): encode_image on the frames after the reference
Preprocessing, encode_text on hand-built SOT ... EOT rows with zero padding.  Only outputs and the inferred configs are stored;
weights and inputs are regenerated from the seeds below.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from univtg_b200 import synth  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_clip.npz")
CONFIGS = ("small224", "small64")
WEIGHT_SEED, FRAME_SEED, TOKEN_SEED = 7, 8, 9
N_FRAMES = 3
TEXT_LENGTHS = (2, 7, 20, 32)  # SOT + words + EOT; 32 is clip.tokenize's max_valid_length
# order of the stored config vector (build_model's CLIP(...) arguments, heads included)
CONFIG_FIELDS = ("embed_dim", "image_resolution", "vision_layers", "vision_width", "patch_size", "vision_heads", "context_length",
                 "vocab_size", "text_width", "text_heads", "text_layers")


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def inferred_config(model):
    v, t = model.visual, model.transformer
    return dict(embed_dim=model.text_projection.shape[1], image_resolution=v.input_resolution, vision_layers=v.transformer.layers,
                vision_width=v.conv1.out_channels, patch_size=v.conv1.kernel_size[0], vision_heads=v.transformer.resblocks[0].attn.num_heads,
                context_length=model.context_length, vocab_size=model.vocab_size, text_width=t.width,
                text_heads=t.resblocks[0].attn.num_heads, text_layers=t.layers)


def main(checkout):
    M = _load(os.path.join(checkout, "run_on_video", "clip", "model.py"), "ref_clip_model")
    pre = _load(os.path.join(checkout, "run_on_video", "preprocessing.py"), "ref_clip_preprocessing").Preprocessing()
    torch.manual_seed(0)
    out = {"text_lengths": np.array(TEXT_LENGTHS, dtype=np.int64), "config_fields": np.array(CONFIG_FIELDS)}
    for name in CONFIGS:
        cfg = synth.CLIP_CONFIGS[name]
        sd = synth.make_clip_state_dict(cfg, seed=WEIGHT_SEED)
        model = M.build_model(dict(sd))  # the reference's own architecture inference (and fp16 conversion)
        inf = inferred_config(model)
        model.float()
        model.load_state_dict({k: v for k, v in sd.items() if k not in ("input_resolution", "context_length", "vocab_size")})
        frames = synth.make_clip_frames(cfg, N_FRAMES, seed=FRAME_SEED)
        # video_loader.py:166-169 (float32, NCHW), then Preprocessing
        images = pre(frames.to(torch.float32).permute(0, 3, 1, 2))
        tokens = synth.make_clip_tokens(cfg, TEXT_LENGTHS, seed=TOKEN_SEED)
        with torch.no_grad():
            img = model.encode_image(images)
            txt = model.encode_text(tokens)
        out[f"{name}/config"] = np.array([inf[f] for f in CONFIG_FIELDS], dtype=np.int64)
        out[f"{name}/image"] = img.numpy().astype(np.float32)
        out[f"{name}/last_hidden_state"] = txt["last_hidden_state"].numpy().astype(np.float32)
        out[f"{name}/pooler_output"] = txt["pooler_output"].numpy().astype(np.float32)
    np.savez(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])

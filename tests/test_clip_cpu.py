"""CLIP feature extraction without a GPU: the fp64 oracle against the reference's own outputs, the architecture inference, the C ABI
surface, loud refusals on the host, and the ptxas record of the new kernels."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import __graft_entry__ as G
from oracle import clip_oracle as CO
from univtg_b200 import _lib, clip, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_clip.npz")
WEIGHT_SEED, FRAME_SEED, TOKEN_SEED, N_FRAMES = 7, 8, 9, 3  # tests/golden/make_golden_clip.py


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def golden_case(z, name):
    cfg = synth.CLIP_CONFIGS[name]
    sd = synth.make_clip_state_dict(cfg, seed=WEIGHT_SEED)
    frames = synth.make_clip_frames(cfg, N_FRAMES, seed=FRAME_SEED)
    tokens = synth.make_clip_tokens(cfg, [int(n) for n in z["text_lengths"]], seed=TOKEN_SEED)
    return cfg, sd, frames, tokens


@pytest.mark.parametrize("name", ["small224", "small64"])
def test_oracle_matches_reference_outputs(golden, name):
    cfg, sd, frames, tokens = golden_case(golden, name)
    img = CO.encode_image(sd, cfg, CO.preprocess(frames))
    txt = CO.encode_text(sd, cfg, tokens)
    for key, got in (("image", img), ("last_hidden_state", txt["last_hidden_state"]), ("pooler_output", txt["pooler_output"])):
        ref = torch.from_numpy(golden[f"{name}/{key}"]).double()
        torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5, msg=lambda m: f"{name} {key}: {m}")


@pytest.mark.parametrize("name", ["small224", "small64"])
def test_config_inference_matches_reference_build_model(golden, name):
    cfg = clip.config_from_state_dict(synth.make_clip_state_dict(synth.CLIP_CONFIGS[name], seed=WEIGHT_SEED))
    mine = dict(cfg, vision_heads=cfg["vision_width"] // 64, text_heads=cfg["text_width"] // 64)
    ref = dict(zip([str(f) for f in golden["config_fields"]], [int(v) for v in golden[f"{name}/config"]]))
    assert mine == ref
    assert cfg == synth.CLIP_CONFIGS[name]


def test_config_inference_of_the_vit_b32_shape():
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    shapes = synth.clip_state_dict_shapes(cfg)
    sd = {k: torch.empty(s, device="meta") for k, s in shapes.items()}
    assert clip.config_from_state_dict(sd) == cfg


def test_resnet_state_dict_is_not_implemented():
    sd = {"visual.layer1.0.conv1.weight": torch.zeros(64, 64, 1, 1), "text_projection": torch.zeros(512, 1024)}
    with pytest.raises(NotImplementedError, match="ModifiedResNet"):
        clip.config_from_state_dict(sd)
    with pytest.raises(NotImplementedError, match="ModifiedResNet"):
        clip.ClipEncoder.from_state_dict(sd)


def test_state_dict_loads_strictly_and_drops_integer_entries():
    cfg = synth.CLIP_CONFIGS["small64"]
    sd = synth.make_clip_state_dict(cfg, seed=1)
    enc = clip.ClipEncoder.from_state_dict(sd)
    assert not enc.training
    assert set(enc.state_dict()) == set(sd) - {"input_resolution", "context_length", "vocab_size"}
    assert len(enc._abi_params()) == 13 + 12 * (cfg["vision_layers"] + cfg["text_layers"])
    half = clip.ClipEncoder.from_state_dict({k: (v.half() if v.is_floating_point() else v) for k, v in sd.items()})
    assert half.text_projection.dtype == torch.float16


def test_abi_symbols_and_host_side_checks():
    lib = _lib.load_library()
    for s in ("univtg_clip_num_params", "univtg_clip_packed_bytes", "univtg_clip_pack_weights", "univtg_clip_workspace_bytes",
              "univtg_clip_encode_image", "univtg_clip_encode_text", "univtg_clip_num_launches"):
        assert hasattr(lib, s) and s in _lib.SIGNATURES
    c = synth.CLIP_CONFIGS["vit_b32"]
    cfg = _lib.ClipConfig(*[c[k] for k in clip.CONFIG_FIELDS], 0)
    assert lib.univtg_clip_num_params(ctypes.byref(cfg)) == 13 + 12 * 24
    pb = lib.univtg_clip_packed_bytes(ctypes.byref(cfg))
    # 16-bit block matrices (12 x 12 W^2 per tower: 84.9 M + 37.7 M) + fp32 token embedding (25.3 M) and the small rest
    assert 2 * 122.6e6 + 4 * 25.2e6 < pb < 2 * 126e6 + 4 * 26e6
    ws = lib.univtg_clip_workspace_bytes(ctypes.byref(cfg), 300, 64, 77)
    assert ws >= 300 * 50 * 768 * 4
    assert lib.univtg_clip_num_launches(ctypes.byref(cfg), 0, 0) == 7 * 12 + 4
    assert lib.univtg_clip_num_launches(ctypes.byref(cfg), 1, 3) == 7 * 12 + 3
    assert lib.univtg_clip_num_launches(ctypes.byref(cfg), 1, 1) == 7 * 12 + 1
    bad = _lib.ClipConfig(*[c[k] for k in clip.CONFIG_FIELDS], 2)
    assert lib.univtg_clip_packed_bytes(ctypes.byref(bad)) == 0
    assert "fp16x3" in _lib.last_error()
    odd = _lib.ClipConfig(*[c[k] if k != "vision_width" else 800 for k in clip.CONFIG_FIELDS], 0)
    assert lib.univtg_clip_num_params(ctypes.byref(odd)) == -1
    assert "vision_width" in _lib.last_error()
    # argument checks run before any device work
    assert lib.univtg_clip_encode_image(ctypes.byref(cfg), None, None, 0, 1, None, 0, None, None) != 0
    assert "packed" in _lib.last_error()
    assert lib.univtg_clip_encode_image(ctypes.byref(cfg), 16, 16, 5, 1, 16, 1 << 40, 16, None) != 0
    assert "pixel_kind" in _lib.last_error()
    assert lib.univtg_clip_encode_image(ctypes.byref(cfg), 16, 16, 0, 2, 16, 100, 16, None) != 0
    assert "ws_bytes" in _lib.last_error()
    assert lib.univtg_clip_encode_text(ctypes.byref(cfg), 16, 16, 1, 78, 16, 1 << 40, 16, None, None) != 0
    assert "ctx_used" in _lib.last_error()
    assert lib.univtg_clip_encode_text(ctypes.byref(cfg), 16, 16, 1, 77, 16, 1 << 40, None, None, None) != 0
    assert "both null" in _lib.last_error()
    for n in (0, 65536):  # one attention grid z-slice per frame / token row
        assert lib.univtg_clip_encode_image(ctypes.byref(cfg), 16, 16, 0, n, 16, 1 << 40, 16, None) != 0
        assert f"n {n} must be in [1, 65535]" in _lib.last_error()
        assert lib.univtg_clip_encode_text(ctypes.byref(cfg), 16, 16, n, 77, 16, 1 << 40, 16, None, None) != 0
        assert f"n {n} must be in [1, 65535]" in _lib.last_error()


def test_entry_points_without_a_gpu_fail_loudly():
    cfg = synth.CLIP_CONFIGS["small64"]
    enc = clip.ClipEncoder.from_state_dict(synth.make_clip_state_dict(cfg, seed=1))
    frames = synth.make_clip_frames(cfg, 2)
    tokens = synth.make_clip_tokens(cfg, [5])
    with pytest.raises(RuntimeError, match="CPU"):
        enc.encode_image(frames)
    with pytest.raises(RuntimeError, match="CPU"):
        enc.encode_text(tokens)
    with pytest.raises(RuntimeError, match="CPU"):
        enc.text_features(tokens)
    with pytest.raises(RuntimeError, match="CUDA"):
        clip.grounding_inputs(torch.zeros(3, 64), torch.zeros(2, 64))
    with pytest.raises(ValueError, match="fp16x3"):
        clip.ClipEncoder(cfg, operand_format="fp16x3")
    with pytest.raises(RuntimeError, match="inference-only"):
        enc.train().encode_image(frames)
    with pytest.raises(ValueError, match="tokens must hold between 1 and 65535 rows per call, got 0"):
        enc.eval().text_features(torch.zeros(0, cfg["context_length"], dtype=torch.int64))


def test_oracle_grounding_inputs_is_load_data():
    g = torch.Generator().manual_seed(0)
    vid, txt = torch.randn(7, 16, generator=g, dtype=torch.float64), torch.randn(4, 16, generator=g, dtype=torch.float64)
    inputs, targets = CO.grounding_inputs(vid, txt)
    v = vid.numpy() / (np.linalg.norm(vid.numpy(), axis=-1, keepdims=True) + 1e-5)
    np.testing.assert_allclose(inputs["src_vid"][0, :, :16].numpy(), v, rtol=1e-12)
    np.testing.assert_allclose(inputs["src_vid"][0, :, 16:].numpy(), np.stack([np.arange(7) / 7, np.arange(7) / 7 + 1 / 7], 1), rtol=1e-12)
    np.testing.assert_allclose(targets["timestamp"][0].numpy(), np.repeat(((np.arange(7) + 1.0) / 7)[:, None], 2, 1), rtol=1e-12)
    assert inputs["src_txt"].shape == (1, 4, 16) and inputs["src_txt_mask"].sum() == 4


# ---- ptxas record of the new kernels (no GPU needed) ----
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


@pytest.fixture(scope="module")
def ptxas_logs():
    if NVCC is None:
        pytest.skip("nvcc not found")
    logs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for src in ("clip.cu", "attention.cu"):
            cmd = [NVCC] + G.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(G.CSRC, src), "-o", os.path.join(tmp, src + ".o")]
            r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            assert r.returncode == 0, r.stdout[-4000:]
            logs[src] = r.stdout
    return logs


def _kernels(log, pattern):
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if re.search(pattern, m.group(1)) else None
            if cur:
                out[cur] = None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = tuple(int(x) for x in m.groups())
    return out


def test_new_kernels_do_not_spill(ptxas_logs):
    k = _kernels(ptxas_logs["clip.cu"], r"\d+clip_(pack|frames|embed|head_ln)_kernel")
    k.update(_kernels(ptxas_logs["attention.cu"], r"attention_wgmma_causal_kernel"))
    assert len(k) == 6, sorted(k)  # pack, frames, embed, head LayerNorm; causal attention fp16 + bf16
    for name, v in k.items():
        assert v is not None and v[1] == 0 and v[2] == 0, (name, v)
    for log in ptxas_logs.values():
        assert "C7511" not in log

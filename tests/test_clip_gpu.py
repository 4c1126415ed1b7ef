"""CLIP feature extraction on the GPU (univtg_b200.clip, csrc/clip.cu) against the fp64 oracle (oracle/clip_oracle.py).

Two bars per output:
  * against the oracle with the kernels' 16-bit operand rounding (opq) - a tight bar on the arithmetic;
  * against the exact fp64 oracle, the error (max and RMS) is no larger than that of the reference's own way of running CLIP on a
    GPU: torch eager with the weights converted to the 16-bit type (convert_weights), computed by the oracle in that dtype.
The oracle runs on the GPU in fp64 so that the ViT-B/32-sized cases stay fast.
"""
import os

import numpy as np
import pytest
import torch

from oracle import clip_oracle as CO
from oracle import univtg_oracle as O
from univtg_b200 import _lib, build_model, clip, synth

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
OPQ = {"fp16": CO.round_fp16, "bf16": CO.round_bf16}
EAGER = {"fp16": torch.float16, "bf16": torch.bfloat16}
# |ours - emulating oracle| <= TIGHT * max|exact| per output
TIGHT = {"fp16": 2e-3, "bf16": 1.5e-2}

_CACHE = {}


def encoder(name, fmt, seed=0):
    key = (name, fmt, seed)
    if key not in _CACHE:
        _CACHE.clear()
        sd = synth.make_clip_state_dict(synth.CLIP_CONFIGS[name], seed=seed)
        _CACHE[key] = (clip.ClipEncoder.from_state_dict(sd, operand_format=fmt).to(DEV), sd)
    return _CACHE[key]


def text_lengths(n, seed):
    g = torch.Generator().manual_seed(seed)
    return [int(x) for x in torch.randint(2, 33, (n,), generator=g)]


def errors(got, ref):
    d = (got.double() - ref.double()).abs()
    return float(d.max()), float(d.pow(2).mean().sqrt())


def check_output(tag, fmt, got, emu, exact, eager):
    scale = float(exact.abs().max())
    e_emu = errors(got, emu)[0]
    ours, base = errors(got, exact), errors(eager, exact)
    print(f"{tag}: vs-emu max {e_emu:.3e} (bar {TIGHT[fmt] * scale:.3e}); vs-exact max {ours[0]:.3e} rms {ours[1]:.3e}; "
          f"torch {fmt} eager max {base[0]:.3e} rms {base[1]:.3e}; ratio max {ours[0] / base[0]:.3f} rms {ours[1] / base[1]:.3f}")
    assert e_emu <= TIGHT[fmt] * scale, f"{tag}: {e_emu} vs emulating oracle"
    assert ours[0] <= base[0] and ours[1] <= base[1], f"{tag}: error {ours} exceeds torch {fmt} eager {base}"


def run_all(enc, sd, cfg, fmt, frames, tokens):
    images = CO.preprocess(frames)
    with torch.no_grad():
        got_i = enc.encode_image(frames)
        got_t = enc.encode_text(tokens)
        ex_i = CO.encode_image(sd, cfg, images)
        ex_t = CO.encode_text(sd, cfg, tokens)
        em_i = CO.encode_image(sd, cfg, images, opq=OPQ[fmt])
        em_t = CO.encode_text(sd, cfg, tokens, opq=OPQ[fmt])
        ea_i = CO.encode_image(sd, cfg, images, dtype=EAGER[fmt])
        ea_t = CO.encode_text(sd, cfg, tokens, dtype=EAGER[fmt])
    return (got_i, got_t), (ex_i, ex_t), (em_i, em_t), (ea_i, ea_t)


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("T,N", [(1, 1), (7, 5), (64, 33)])
def test_vit_b32_against_oracle_and_torch_eager(fmt, T, N):
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    enc, sd = encoder("vit_b32", fmt)
    frames = synth.make_clip_frames(cfg, T, seed=T).to(DEV)
    tokens = synth.make_clip_tokens(cfg, text_lengths(N, N), seed=N).to(DEV)
    got, ex, em, ea = run_all(enc, sd, cfg, fmt, frames, tokens)
    check_output(f"vit_b32 {fmt} T={T} image", fmt, got[0], em[0], ex[0], ea[0])
    for k in ("last_hidden_state", "pooler_output"):
        check_output(f"vit_b32 {fmt} N={N} {k}", fmt, got[1][k], em[1][k], ex[1][k], ea[1][k])


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("name", ["small224", "small64"])
def test_small_configs_against_reference_goldens(golden_dir, name, fmt):
    z = dict(np.load(os.path.join(golden_dir, "reference_clip.npz")))
    cfg = synth.CLIP_CONFIGS[name]
    enc, sd = encoder(name, fmt, seed=7)
    frames = synth.make_clip_frames(cfg, 3, seed=8).to(DEV)
    tokens = synth.make_clip_tokens(cfg, [int(n) for n in z["text_lengths"]], seed=9).to(DEV)
    got, ex, em, ea = run_all(enc, sd, cfg, fmt, frames, tokens)
    ref = {k: torch.from_numpy(z[f"{name}/{k}"]).to(DEV) for k in ("image", "last_hidden_state", "pooler_output")}
    check_output(f"{name} {fmt} image", fmt, got[0], em[0], ref["image"], ea[0])
    for k in ("last_hidden_state", "pooler_output"):
        check_output(f"{name} {fmt} {k}", fmt, got[1][k], em[1][k], ref[k], ea[1][k])


def test_causality_is_bit_exact():
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    enc, _ = encoder("vit_b32", "fp16")
    tokens = synth.make_clip_tokens(cfg, [12, 30, 5], seed=3).to(DEV)
    base = enc.encode_text(tokens)
    for j in (0, 4, 11):  # inside row 0 (EOT at 11)
        t2 = tokens.clone()
        t2[0, j] = 1234 if int(t2[0, j]) != 1234 else 4321
        out = enc.encode_text(t2)
        assert torch.equal(out["last_hidden_state"][0, :j], base["last_hidden_state"][0, :j])
        assert torch.equal(out["last_hidden_state"][1:], base["last_hidden_state"][1:])
        assert not torch.equal(out["last_hidden_state"][0, j:], base["last_hidden_state"][0, j:])
    t2 = tokens.clone()
    t2[0, 20] = 777  # after EOT: pooled (EOT row) and every row < 20 unchanged
    out = enc.encode_text(t2)
    assert torch.equal(out["last_hidden_state"][0, :20], base["last_hidden_state"][0, :20])
    assert torch.equal(out["pooler_output"], base["pooler_output"])


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_uint8_and_normalised_float_inputs_agree(fmt):
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    enc, _ = encoder("vit_b32", fmt)
    frames = synth.make_clip_frames(cfg, 5, seed=11).to(DEV)
    a = enc.encode_image(frames)
    # Preprocessing on the host in fp32, where the reference's loader runs it (torch's CUDA division by a scalar multiplies by the
    # reciprocal instead, which moves some inputs by an ulp and then flips their 16-bit rounding)
    b = enc.encode_image(CO.preprocess(frames.cpu()).to(DEV))
    # both forms reach the kernels as the same fp32 values, rounded once to the operand format
    assert torch.equal(a, b), float((a - b).abs().max())


def test_a_frame_alone_agrees_with_the_same_frame_in_a_batch():
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    enc, _ = encoder("vit_b32", "fp16")
    frames = synth.make_clip_frames(cfg, 40, seed=12).to(DEV)
    batch = enc.encode_image(frames)
    for i in (0, 17, 39):
        alone = enc.encode_image(frames[i:i + 1])
        torch.testing.assert_close(alone[0], batch[i], rtol=0, atol=1e-5 * float(batch.abs().max()))


def test_batches_beyond_one_row_per_warp_of_a_capped_grid():
    """More stream rows than the row kernels' grid has warps (65536 blocks x 8 warps = 524288): the last frames and token rows of
    a large batch equal the same inputs encoded in a small batch."""
    cfg = synth.CLIP_CONFIGS["small64"]  # 17 tokens per frame
    enc, _ = encoder("small64", "fp16")
    small = synth.make_clip_frames(cfg, 8, seed=14).to(DEV)
    n = 31000  # 527000 stream rows
    big = small.repeat(n // 8 + 1, 1, 1, 1)[:n].contiguous()
    ref = enc.encode_image(small)
    out = enc.encode_image(big)
    for i in (0, n - 9, n - 2, n - 1):
        torch.testing.assert_close(out[i], ref[i % 8], rtol=0, atol=1e-5 * float(ref.abs().max()))
    tokens = synth.make_clip_tokens(cfg, [5, 9, 32, 17], seed=15).to(DEV)
    m = 6812  # 524524 rows of 77 positions
    big_t = tokens.repeat(m // 4, 1).contiguous()
    ref_t = enc.encode_text(tokens)
    out_t = enc.encode_text(big_t)
    for i in (0, m - 3, m - 1):
        for k in ("last_hidden_state", "pooler_output"):
            torch.testing.assert_close(out_t[k][i], ref_t[k][i % 4], rtol=0, atol=1e-5 * float(ref_t[k].abs().max()))


def test_text_features_are_the_valid_rows_of_encode_text():
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    enc, _ = encoder("vit_b32", "fp16")
    lengths = [9, 32, 3, 17]
    tokens = synth.make_clip_tokens(cfg, lengths, seed=13).to(DEV)
    full = enc.encode_text(tokens)["last_hidden_state"]
    feats, mask = enc.text_features(tokens)
    assert feats.shape == (4, 32, cfg["text_width"]) and mask.shape == (4, 32)
    assert mask.sum(1).tolist() == [float(n) for n in lengths]
    for i, n in enumerate(lengths):
        torch.testing.assert_close(feats[i, :n], full[i, :n], rtol=0, atol=1e-5 * float(full.abs().max()))
        assert torch.count_nonzero(feats[i, n:]) == 0


def test_launch_counter_matches_num_launches():
    cfg = synth.CLIP_CONFIGS["small64"]
    enc, _ = encoder("small64", "fp16")
    frames = synth.make_clip_frames(cfg, 4).to(DEV)
    tokens = synth.make_clip_tokens(cfg, [5, 9]).to(DEV)
    enc.encode_image(frames)  # packs the weights
    lib = _lib.load_library()
    for call, n in ((lambda: enc.encode_image(frames), enc.num_launches(0)),
                    (lambda: enc.encode_text(tokens), enc.num_launches(1, 3)),
                    (lambda: enc.text_features(tokens), enc.num_launches(1, 1))):
        c0 = lib.univtg_launch_count()
        call()
        assert lib.univtg_launch_count() - c0 == n
    assert enc.num_launches(0) == 7 * cfg["vision_layers"] + 4


def test_refusals_launch_nothing():
    cfg = synth.CLIP_CONFIGS["small64"]
    enc, sd = encoder("small64", "fp16")
    tokens = synth.make_clip_tokens(cfg, [5, 9]).to(DEV)
    enc.encode_text(tokens)  # packs the weights
    lib = _lib.load_library()
    c0 = lib.univtg_launch_count()
    bad = tokens.clone()
    bad[1, 3] = cfg["vocab_size"]
    with pytest.raises(RuntimeError, match=r"tokens\[1, 3\] = 49408 is outside"):
        enc.encode_text(bad)
    bad[1, 3] = -1
    with pytest.raises(RuntimeError, match="outside"):
        enc.text_features(bad)
    with pytest.raises(RuntimeError, match="CPU"):
        enc.encode_image(synth.make_clip_frames(cfg, 1))
    with pytest.raises(RuntimeError, match="CPU"):
        enc.encode_text(tokens.cpu())
    with pytest.raises(ValueError, match="fp16x3"):
        clip.ClipEncoder.from_state_dict(sd, operand_format="fp16x3")
    resnet = {"visual.layer1.0.conv1.weight": torch.zeros(64, 64, 1, 1, device=DEV)}
    with pytest.raises(NotImplementedError, match="ModifiedResNet"):
        clip.ClipEncoder.from_state_dict(resnet)
    with pytest.raises(RuntimeError, match="inference-only"):
        enc.train().encode_text(tokens)
    enc.eval()
    assert lib.univtg_launch_count() == c0


def test_end_to_end_frames_and_query_to_grounding():
    """Frames + query tokens -> CLIP -> grounding_inputs -> a cfg1-shaped UniVTG model (v_feat_dim 514 = 512 + 2 TEF, t_feat_dim 512)
    -> decode_mr, against the same pipeline on the fp64 oracles, at the cfg1 bars."""
    from univtg_b200 import postproc

    ccfg = synth.CLIP_CONFIGS["vit_b32"]
    ucfg = synth.CONFIGS["cfg1"]
    enc, csd = encoder("vit_b32", "fp16")
    frames = synth.make_clip_frames(ccfg, ucfg["l_vid"], seed=21).to(DEV)
    tokens = synth.make_clip_tokens(ccfg, [ucfg["l_txt"]], seed=22).to(DEV)
    model, _ = build_model(synth.reference_args(ucfg, device=DEV))
    usd = synth.make_state_dict(ucfg, seed=23)
    model.load_state_dict(usd, strict=True)
    model.to(DEV).eval()
    with torch.no_grad():
        vid = enc.encode_image(frames)
        txt, mask = enc.text_features(tokens)
        inputs, targets = clip.grounding_inputs(vid, txt[0][mask[0] > 0])
        out = model(**inputs)
        windows = postproc.decode_mr(out, targets, None)
        ovid = CO.encode_image(csd, ccfg, CO.preprocess(frames))
        otxt = CO.encode_text(csd, ccfg, tokens)["last_hidden_state"][0, :ucfg["l_txt"]]
        oin, otg = CO.grounding_inputs(ovid, otxt)
    oin = {k: v.cpu() for k, v in oin.items()}
    ref = O.forward(usd, ucfg, **oin)
    assert inputs["src_vid"].shape == (1, ucfg["l_vid"], 514) and inputs["src_txt"].shape == (1, ucfg["l_txt"], 512)
    torch.testing.assert_close(targets["timestamp"].double().cpu(), otg["timestamp"].cpu())
    for k in ("pred_logits", "pred_spans", "saliency_scores"):
        torch.testing.assert_close(out[k].double().cpu(), ref[k], rtol=1e-3, atol=1e-4, msg=lambda m: f"end to end {k}: {m}")
    assert windows["windows"].shape == (1, ucfg["l_vid"], 3)

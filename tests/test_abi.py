"""The C-ABI library loads (no GPU needed) and exports every symbol include/univtg_b200.h declares."""
import ctypes
import os
import re

from univtg_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "univtg_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(univtg_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load_library()
    syms = _declared_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/univtg_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature in univtg_b200/_lib.py"


def test_abi_version_and_sizes():
    lib = _lib.load_library()
    assert lib.univtg_abi_version() == 2
    cfg = _lib.Config(1024, 8, 1024, 4, 2, 2818, 512, 0)
    assert lib.univtg_num_params(ctypes.byref(cfg)) == 8 * 2 + 1 + 12 * 4 + 12 + 1
    pb = lib.univtg_packed_bytes(ctypes.byref(cfg))
    # 16-bit copies of every GEMM weight (K padded to 64) + fp32 vectors: between 2 and 2.3 bytes per used parameter
    assert 2.0 * 43.3e6 < pb < 2.3 * 43.3e6
    shp = _lib.Shape(32, 75, 32, 0)
    assert lib.univtg_workspace_bytes(ctypes.byref(cfg), ctypes.byref(shp)) > 50e6


def test_bad_config_is_rejected_with_message():
    lib = _lib.load_library()
    cfg = _lib.Config(1000, 8, 1024, 4, 2, 2818, 512, 0)
    assert lib.univtg_packed_bytes(ctypes.byref(cfg)) == 0
    assert "hidden_dim" in _lib.last_error()


def test_tile_cost_model_choices_are_legal_and_sensible():
    """Host-side launch planning (choose_tile, gemm.cu): legal tile widths / split factors, single-round tilings when they
    exist, split-K for weight-gradient shapes (few output tiles, long K)."""
    import ctypes

    from univtg_b200 import _lib

    lib = _lib.load_library()

    def choose(problems, step, max_split, sms=132):
        n = len(problems)
        Ms = (ctypes.c_int32 * n)(*[p[0] for p in problems])
        Ns = (ctypes.c_int32 * n)(*[p[1] for p in problems])
        kb = (ctypes.c_int32 * n)(*[(p[2] + 63) // 64 for p in problems])
        bn, ks = ctypes.c_int32(0), ctypes.c_int32(0)
        assert lib.univtg_debug_choose_tile(Ms, Ns, kb, n, sms, step, max_split, ctypes.byref(bn), ctypes.byref(ks)) == 0
        return bn.value, ks.value

    M, d, Mh = 3424, 1024, 2432
    for problems, step, max_split in ([[(M, d, d)], 16, 1], [[(M, 2 * d, d), (M, d, d)], 16, 1], [[(Mh, 2 * d, 3 * d)], 16, 1],
                                      [[(d, d, M)], 64, 16], [[(2 * d, d, M), (d, d, M)], 64, 16], [[(d, d, Mh)] * 3, 64, 8],
                                      [[(300, 384, 200)], 16, 1], [[(64, 64, 64)], 64, 16]):
        bn, ks = choose(problems, step, max_split)
        assert 64 <= bn <= 256 and bn % step == 0
        assert 1 <= ks <= max_split and (ks & (ks - 1)) == 0
        assert ks == 1 or all(ks * 4 <= (p[2] + 63) // 64 for p in problems)
    # N = 1024 over 27 row tiles: a single round exists (<= 132 tiles on H100) and must be chosen
    bn, ks = choose([(M, d, d)], 16, 1)
    assert ((M + 127) // 128) * ((d + bn - 1) // bn) <= 132 and ks == 1
    # weight gradient d x d with K = 3424: 32 output tiles -> split-K so that most SMs work
    bn, ks = choose([(d, d, M)], 64, 16)
    assert bn == 256 and ks >= 2 and 8 * 4 * ks <= 132
    # bad arguments are rejected
    z = ctypes.c_int32(0)
    assert lib.univtg_debug_choose_tile(None, None, None, 1, 132, 16, 1, ctypes.byref(z), ctypes.byref(z)) != 0


def test_product_entry_points_fail_loudly_without_cuda():
    """No CPU / eager fallback anywhere on the product path: every host-side entry point raises on CPU tensors / models."""
    import pytest
    import torch

    from univtg_b200 import build_model, postproc, synth
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS["tiny"]
    model, crit = build_model(synth.reference_args(cfg, device="cpu"))
    inp = synth.make_inputs(cfg, seed=1, ragged=True, batch=2)
    tgt = synth.make_targets(inp, seed=2)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.eval()
        model(**inp)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.train()
        model(**inp)
    B, Lv = inp["src_vid"].shape[:2]
    fake = {"pred_logits": torch.rand(B, Lv, 1), "pred_spans": torch.rand(B, Lv, 2), "vid_mem_proj": torch.rand(B, Lv, cfg["hidden_dim"]),
            "txt_mem_proj": torch.rand(B, 1, cfg["hidden_dim"]), "saliency_scores": torch.rand(B, Lv), "src_vid_mask": inp["src_vid_mask"]}
    with pytest.raises(RuntimeError, match="CUDA"):
        crit(fake, tgt)
    with pytest.raises(RuntimeError, match="CUDA"):
        postproc.decode_mr(fake, {"timestamp": tgt["timestamp"], "timestamp_mask": tgt["timestamp_mask"]}, [10.0] * B)
    with pytest.raises(RuntimeError, match="CUDA"):
        postproc.temporal_nms(torch.zeros(B, 4, 3, dtype=torch.float64), 0.5)
    with pytest.raises(RuntimeError, match="CUDA"):
        FlatAdamW(model)

"""The fp16x3 operand format can reach the strict mode's bars: the fp64 oracle, with every tensor-core operand rounded to an
fp16 hi / lo pair, against the fp32 reference outputs."""
import pytest
import torch

from oracle import univtg_oracle as O
from tests.helpers import GOLDEN_CASES, golden_out, load_golden, subsample
from tests.strict_oracle import round_fp16x3

# Shared with tests/test_strict_gpu.py.
HEAD_TOL = dict(rtol=2e-5, atol=2e-6)   # pred_logits, pred_spans, saliency_scores
PROJ_TOL = dict(rtol=1e-4, atol=1e-5)   # vid_mem_proj, txt_mem_proj
ARGMAX_MARGIN = 1e-5


def check_against_reference(out, z, name, proj=PROJ_TOL):
    for k in ("pred_logits", "pred_spans", "saliency_scores"):
        torch.testing.assert_close(out[k].double().cpu(), golden_out(z, k).double(), **HEAD_TOL, msg=lambda m: f"{name}/{k}: {m}")
    torch.testing.assert_close(subsample("vid_mem_proj", out["vid_mem_proj"].double().cpu(), z), golden_out(z, "vid_mem_proj").double(),
                               **proj, msg=lambda m: f"{name}/vid_mem_proj: {m}")
    torch.testing.assert_close(out["txt_mem_proj"].double().cpu(), golden_out(z, "txt_mem_proj").double(), **proj,
                               msg=lambda m: f"{name}/txt_mem_proj: {m}")
    for k, got in (("pred_logits", out["pred_logits"].cpu().squeeze(-1)), ("saliency_scores", out["saliency_scores"].cpu())):
        ref = golden_out(z, k)
        ref = ref.squeeze(-1) if ref.dim() == 3 else ref
        t2 = ref.topk(2, dim=1).values
        dec = (t2[:, 0] - t2[:, 1]) > ARGMAX_MARGIN
        assert torch.equal(got.argmax(1)[dec], ref.argmax(1)[dec]), f"{name}/{k}: argmax differs where the margin exceeds 1e-5"


def test_round_fp16x3_is_a_split_pair():
    x = torch.randn(4096, dtype=torch.float64) * 3
    r = round_fp16x3(x)
    hi = x.to(torch.float16).double()
    assert torch.equal(r - hi, (x - hi).to(torch.float16).double())
    assert ((r - x).abs() <= 2.0 ** -22 * x.abs() + 2.0 ** -25).all()


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_fp16x3_oracle_meets_strict_bars(name):
    cfg, sd, inp, tgt, z = load_golden(name)
    out = O.forward(sd, cfg, **inp, opq=round_fp16x3)
    check_against_reference(out, z, name)

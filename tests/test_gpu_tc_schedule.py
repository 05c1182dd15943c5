"""Tile-schedule edge cases of the TMA conv kernel: two consumer warpgroups take alternate whole tiles of a CTA's sequence
(132 persistent CTAs on an H100 SXM), so the cases below give one warpgroup no tile, one tile more than the other, and odd tile
counts per CTA at every N tile width.  Checked against torch CPU fp32 with the tolerance of test_gpu_tc.py (bf16x3 split: 1e-4
of the output scale)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ACTS = {0: lambda x: x, 1: F.relu, 2: F.gelu, 3: F.silu}

SCHEDULE_CASES = [
    # n, cin, h, w, cout, k, pad, mode, act   (stride 1; BN is chosen per launch by choose_bn)
    (1, 64, 8, 16, 32, 1, 0, "zeros", 0),           # a single tile: the second warpgroup gets none
    (1, 64, 133, 128, 32, 1, 0, "zeros", 1),        # 133 tiles: one CTA runs two, the others one
    (1, 64, 265, 128, 32, 1, 0, "zeros", 2),        # 265 tiles: one CTA runs three (warpgroup 0 gets one more), BN = 32
    (1, 64, 265, 128, 64, 3, 1, "zeros", 0),        # BN = 64, odd tile count per CTA
    (1, 64, 265, 128, 96, 3, 1, "reflect", 1),      # BN = 96, odd tile count per CTA
    (1, 64, 331, 128, 128, 3, 1, "zeros", 3),       # BN = 128, odd tile count per CTA
]


@pytest.fixture(scope="module")
def eng():
    from mit_b200.engine import get_engine
    e = get_engine("cuda:0")
    e.set_tensor_cores(True)
    yield e
    e.set_tensor_cores(True)


@pytest.mark.parametrize("case", SCHEDULE_CASES)
def test_tma_tile_schedule_matches_fp32(eng, case):
    n, cin, h, w, cout, k, pad, mode, act = case
    g = torch.Generator().manual_seed(1000 + SCHEDULE_CASES.index(case))
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    xp = F.pad(x, (pad, pad, pad, pad), mode="reflect") if mode == "reflect" and pad else x
    ref = ACTS[act](F.conv2d(xp, wt, b, padding=0 if mode == "reflect" else pad))
    eng.profile(True)
    y = eng.conv2d(x, wt, b, (1, 1), (pad, pad), mode, act).cpu()
    rep = eng.profile_report()
    eng.profile(False)
    assert rep.get("conv_tc", {}).get("launches", 0) >= 1, f"tensor-core kernel was not used: {rep}"
    scale = max(1.0, ref.abs().max().item())
    err = (y - ref).abs().max().item()
    assert err <= 1e-4 * scale, f"case {case}: err {err:.3e}"

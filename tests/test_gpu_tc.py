"""The wgmma (bf16x3 operand split) convolution against torch CPU fp32 and against the exact-fp32 SIMT kernel.
Tolerance: the split drops terms of <= ~3*2^-18 relative per product -> 1e-4 of the output scale is a safe bound
(observed ~1e-6..1e-5); the networks' 1e-3 budget is checked in test_gpu_nets.py with tensor cores on."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)


@pytest.fixture(scope="module")
def eng():
    from mit_b200.engine import get_engine
    e = get_engine("cuda:0")
    yield e
    e.set_tensor_cores(True)


ACTS = {0: lambda x: x, 1: F.relu, 2: F.gelu, 3: F.silu, 4: torch.sigmoid}

TC_CASES = [
    # n, cin, h, w, cout, k, stride, pad, mode, act   (all eligible: cin % 8 == 0, cout >= 16)
    (1, 64, 16, 16, 128, 1, 1, 0, "zeros", 0),         # one K block, one tile
    (1, 128, 20, 24, 256, 1, 1, 0, "zeros", 2),        # two N tiles of 128
    (2, 128, 12, 20, 512, 1, 1, 0, "zeros", 2),        # two N tiles
    (1, 512, 9, 13, 128, 3, 1, 1, "reflect", 1),       # LaMa to_l: K = 4608 (72 K blocks, pipeline wrap-around)
    (1, 128, 17, 23, 384, 3, 1, 1, "reflect", 0),      # three N tiles of 128
    (1, 40, 24, 50, 80, 3, 1, 1, "zeros", 0),          # OCR layer1: Cin = 40 (chunks straddle K blocks, not taps)
    (1, 320, 6, 33, 320, 3, (2, 1), 1, "zeros", 0),    # N padded to 3 tiles of 128, stride (2,1)
    (1, 256, 14, 10, 128, 7, 1, 3, "zeros", 0),        # dense 7x7
    (1, 64, 31, 29, 128, 3, 2, 1, "reflect", 1),       # stride 2, M tail (not a multiple of 128)
    (1, 128, 8, 8, 32, 3, 1, 1, "zeros", 3),           # BN = 32
    (3, 1024, 4, 6, 1024, 2, 2, 0, "zeros", 0),        # downsample conv, 4 N tiles, split-K (16 splits)
    (1, 1024, 12, 16, 128, 7, 1, 3, "zeros", 0),       # DBNet upconv1-like: M = 192, K = 50176 -> split-K
    (1, 64, 40, 36, 3, 3, 1, 1, "reflect", 4),         # thin output on the tensor cores (BN = 32)
    (1, 32, 30, 26, 1, 1, 1, 0, "zeros", 4),           # mask head 1x1 -> 1 channel
    (1, 160, 13, 21, 160, 3, 1, 1, "zeros", 1),        # OCR layer3: Cin = 160 -> per-tap padding to 192 on the TMA path
    (2, 80, 9, 70, 96, 3, 1, 1, "zeros", 0),           # Cin = 80 -> 128, Cout = 96 (BN chosen per launch), batch of 2 patches
    (1, 256, 33, 47, 256, 3, 2, 1, "reflect", 0),      # LaMa downsample: stride 2 + reflect halo through TMA element strides
    (1, 192, 40, 24, 384, 1, 1, 0, "zeros", 0),        # 1x1 on the flattened pixel matrix, M tail
]


@pytest.mark.parametrize("case", TC_CASES)
def test_tc_conv_matches_fp32(eng, case):
    n, cin, h, w, cout, k, stride, pad, mode, act = case
    stride = stride if isinstance(stride, tuple) else (stride, stride)
    g = torch.Generator().manual_seed(abs(hash(case)) % (2 ** 31))
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    xp = F.pad(x, (pad, pad, pad, pad), mode="reflect") if mode == "reflect" and pad else x
    ref = ACTS[act](F.conv2d(xp, wt, b, stride=stride, padding=0 if mode == "reflect" else pad))
    eng.set_tensor_cores(True)
    eng.profile(True)
    y_tc = eng.conv2d(x, wt, b, stride, (pad, pad), mode, act).cpu()
    rep = eng.profile_report()
    eng.profile(False)
    assert rep.get("conv_tc", {}).get("launches", 0) >= 1, f"tensor-core kernel was not used: {rep}"
    eng.set_tensor_cores(False)
    y_simt = eng.conv2d(x, wt, b, stride, (pad, pad), mode, act).cpu()
    eng.set_tensor_cores(True)
    scale = max(1.0, ref.abs().max().item())
    e_tc, e_simt = (y_tc - ref).abs().max().item(), (y_simt - ref).abs().max().item()
    print(f"case {case}: tc err {e_tc:.2e}  simt err {e_simt:.2e}  scale {scale:.2f}")
    assert e_simt <= 2e-4 * scale
    assert e_tc <= 1e-4 * scale, f"tc err {e_tc:.3e}"


def test_tc_conv_prologue_and_transposed(eng):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 80, 12, 37, generator=g)
    wt = torch.randn(160, 80, 3, 3, generator=g) / 27
    sc, sh = torch.rand(80, generator=g) + 0.5, torch.randn(80, generator=g) * 0.3
    ref = F.conv2d(F.relu(x * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)), wt, padding=1)
    eng.set_tensor_cores(True)
    y = eng.conv2d(x, wt, None, (1, 1), (1, 1), "zeros", 0, sc, sh, True).cpu()
    assert (y - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
    for (k, pad, op, cin, cout) in ((2, 0, 0, 64, 64), (4, 1, 0, 32, 32), (3, 1, 1, 128, 64)):
        x = torch.randn(2, cin, 11, 14, generator=g)
        wt = torch.randn(cin, cout, k, k, generator=g) / (cin * k * k / 4) ** 0.5
        b = torch.randn(cout, generator=g)
        ref = F.conv_transpose2d(x, wt, b, stride=2, padding=pad, output_padding=op)
        y = eng.conv_transpose2d(x, wt, b, k, pad, op, 0).cpu()
        assert (y - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item()), (k, pad, op)

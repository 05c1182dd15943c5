"""Edge cases of the TMA conv kernel's staged epilogue (conv_tma.cu: epilogue_staged), checked as tests/test_gpu_conv_epilogue.py
checks the fused epilogue: within the float64-propagated error bound, the NaN sentinel intact outside the written slice, and the
split output (out_sv) bit for bit against the split of out.

The staged epilogue passes a tile through shared memory 32 columns at a time and gives each thread 4 channels (16-byte operands)
or 2 (8-byte operands).  These cases reach what the main module does not: Cout that ends inside a chunk (40, 80, as the bench's
networks have), the 8-byte variant (a channel slice, a residual or a column vector 8- but not 16-byte aligned, Cout not a
multiple of 4), and an edge tile with fewer than 128 valid rows whose add1 is the output itself.  The kernel stages the epilogue
only where the register epilogue would not hide behind the main loop (conv_tma.cu: stage_epilogue), so long-K cases check that
the same float2 outputs still run through the register epilogue.  Every case asserts which of the three ran."""
import pytest
import torch

from test_gpu_conv_epilogue import ALL, GELU, NONE, RELU, SILU, SENT16, Conv, eng, expect_path, host_split, launch, out_sv_buffers, spec  # noqa: F401

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

CASES = [
    # Cout ends inside the N tile's last 32-column chunk
    dict(ALL, cout=40, bn=64, act=GELU, k=1, staged=4),
    dict(ALL, cout=40, bn=64, act=RELU, k=3, staged=4),
    dict(ALL, cout=80, bn=96, act=NONE, k=1, staged=4),
    dict(ALL, cout=80, bn=64, act=SILU, k=3, staged=4),
    # 8-byte operands: out slice at coff 2 (mod 4), add1 slice at coff 6, Cout 202, scale 8- but not 16-byte aligned
    dict(ALL, out_cs=206, out_coff=2, act=GELU, k=1, bn=128, staged=2),
    dict(ALL, add1=dict(cs=210, coff=6), act=RELU, k=3, bn=64, staged=2),
    dict(ALL, cout=202, act=NONE, k=1, bn=96, staged=2),
    dict(ALL, cout=80, scale8=True, act=GELU, k=3, bn=32, staged=2),
    # edge tiles (M = 240: the second 128-row tile has 112 valid rows; k = 3: 32 x 4 patches partly outside the image), add1 == out
    dict(scale=True, mul1=True, add1_out=True, act=GELU, k=1, bn=128, staged=4),
    dict(scale=True, add0=True, add1_out=True, act=RELU, k=3, bn=64, staged=4),
    dict(scale=True, add1_out=True, cout=40, act=NONE, k=1, bn=64, out_cs=44, out_coff=2, staged=2),
    # long K (Cin 512, 3x3: 72 K blocks) over enough tiles not to need split-K: the main loop hides the register epilogue, which
    # runs instead
    dict(ALL, cin=512, h=96, w=96, act=GELU, bn=128, staged=0),
    dict(scale=True, add1_out=True, cin=512, h=96, w=96, cout=40, act=RELU, bn=64, staged=0),
]


def conv(kw, seed):
    kw = dict(kw)
    scale8 = kw.pop("scale8", False)
    staged = kw.pop("staged")
    s = spec(**kw, vec2=1)
    s["staged"] = staged
    c = Conv(s, seed)
    if scale8:                                     # the same scale vector, 8 bytes past a 16-byte boundary
        b = torch.zeros(c.scale.numel() + 2, device="cuda")
        b[2:].copy_(c.scale)
        c.keep.append(b)
        c.d.scale = b.data_ptr() + 8
    return s, c


def run(eng, c, s):
    info = launch(eng, c.d)
    expect_path(s, info)
    assert info.staged == s["staged"], f"staged = {info.staged}, expected {s['staged']}"
    return info


@pytest.mark.parametrize("i", range(len(CASES)))
def test_staged_epilogue(eng, i):
    s, c = conv(CASES[i], 7000 + i)
    info = run(eng, c, s)
    ref, bound = c.reference(info)
    c.check_out(ref, bound, f"staged case {i}")


SV_CASES = [
    dict(ALL, cout=40, bn=64, act=GELU, k=3, staged=4),                    # partial chunk, 16-byte path
    dict(ALL, cout=80, scale8=True, bn=96, act=RELU, k=1, staged=2),       # partial chunk, 8-byte path
    dict(scale=True, add1_out=True, act=RELU, k=1, bn=128, staged=4),      # edge tile, add1 == out
]


@pytest.mark.parametrize("i", range(len(SV_CASES)))
def test_staged_out_sv(eng, i):
    s, c = conv(SV_CASES[i], 7100 + i)
    hi, mid, inside = out_sv_buffers(c, 264, 64, 1)
    info = run(eng, c, s)
    ref, bound = c.reference(info)
    c.check_out(ref, bound, f"staged out_sv case {i}")
    hic, midc = hi.cpu(), mid.cpu()
    assert torch.all(hic[~inside] == SENT16) and torch.all(midc[~inside] == SENT16), "out_sv: write outside the interior slice"
    sl = (slice(None), slice(1, 1 + c.Ho), slice(1, 1 + c.Wo), slice(64, 64 + s["cout"]))
    want_hi, want_mid = host_split(c.y().to(torch.float32))
    assert torch.equal(hic[sl].permute(0, 3, 1, 2), want_hi) and torch.equal(midc[sl].permute(0, 3, 1, 2), want_mid), \
        "out_sv: hi / mid differ from the split of out"

"""Epilogue signatures of the TMA conv kernel's staged epilogue (conv_tma.cu: MITB_EPI_SIGS, epilogue_staged): a staged launch whose
(activation, chain parts) pair has a kernel of its own runs it, with only those parts declared, loaded and applied, and more rows in
flight.  Every instantiated signature is run here at every N tile (BN 32 / 64 / 96 / 128) and both widths of the staged epilogue
(4 channels per thread, and 2 where the output slice is only 8-byte aligned), twice through the test hook: specialised and forced
onto the generic signature (mitb_set_epi_specialise(0)).  The two must agree bit for bit in the fp32 output and in the bf16 hi / mid
operands, and agree with the float64 reference of tests/test_gpu_conv_epilogue.py within its bound.  The cases have an N tail
(Cout 200), a ragged last M tile (240 rows; 3x3 cases: 32 x 4 patches partly outside the image), add1 aliasing the output where
the signature writes one, channel slices, and the split output at a channel offset of a halo'd tensor."""
import ctypes as C

import pytest
import torch

from test_gpu_conv_epilogue import SENT16, SENT32, Conv, eng, expect_path, host_split, launch, out_sv_buffers, spec, split_value, ulp32  # noqa: F401

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

ADD0, SCALE, SHIFT, MUL1, ADD1, OUT, OS, OS_AFFINE, OS_RELU, GENERIC = 1, 2, 4, 8, 16, 32, 64, 128, 256, 512


def signatures():
    from mit_b200 import _lib as L
    lib = L.load()
    n = lib.mitb_test_epi_signatures(None, None, 0)
    act, sig = (C.c_int * n)(), (C.c_int * n)()
    assert lib.mitb_test_epi_signatures(act, sig, n) == n
    return list(zip(act, sig))


SIGS = signatures()
# a split output needs 4-aligned channel pitches and offsets on every operand (launch_conv_tma): its signatures run 4 channels only
CASES = [(a, s, bn, w) for a, s in SIGS for bn in (32, 64, 96, 128) for w in ((4,) if s & OS else (4, 2))]


def set_specialise(eng, on):
    return eng.lib.mitb_set_epi_specialise(on)


def make(act, sig, bn, w, seed):
    kw = dict(act=act, bn=bn, cin=64, cout=200, h=12, w=20, k=1 if (bn // 32 + w) % 2 else 3, shift=bool(sig & SHIFT),
              scale=bool(sig & SCALE), mul1=bool(sig & MUL1), add0=True if sig & ADD0 else None, vec2=1)
    if sig & ADD1:
        kw["add1_out" if sig & OUT else "add1"] = True
    if w == 2:                                 # an output slice 8- but not 16-byte aligned
        kw.update(out_cs=206, out_coff=2)
    s = spec(**kw)
    c = Conv(s, seed)
    sv = None
    if sig & OS:
        sv = out_sv_buffers(c, 264, 64, 1)
        g = torch.Generator().manual_seed(seed + 1)
        if sig & OS_AFFINE:                    # power-of-two scales: fmaf(v, s, t) rounds like the float32 host expression
            c.os_s = (2.0 ** torch.randint(-2, 3, (200,), generator=g)).float() * torch.sign(torch.randn(200, generator=g))
            c.os_t = torch.randn(200, generator=g)
            c.d.os_scale, c.d.os_shift, c.d.os_relu = c.dev(c.os_s), c.dev(c.os_t), int(bool(sig & OS_RELU))
    if not sig & OUT:
        c.d.out = None
    return s, c, sv


def run(eng, c, sv, on, out0):
    c.out.copy_(out0)                          # the sentinel, and add1's values where it aliases the output
    if sv:
        sv[0].fill_(SENT16)
        sv[1].fill_(SENT16)
    prev = set_specialise(eng, on)
    try:
        info = launch(eng, c.d)
    finally:
        set_specialise(eng, prev)
    return info, c.out.clone(), (sv[0].clone(), sv[1].clone()) if sv else None


@pytest.mark.parametrize("i", range(len(CASES)))
def test_signature_matches_generic(eng, i):
    act, sig, bn, w = CASES[i]
    s, c, sv = make(act, sig, bn, w, 8000 + i)
    out0 = c.out.clone()
    info_g, out_g, hm_g = run(eng, c, sv, 0, out0)
    info, out, hm = run(eng, c, sv, 1, out0)
    expect_path(s, info)
    assert info.staged == w and info_g.staged == w, f"staged = {info.staged} / {info_g.staged}, expected {w}"
    assert info_g.epi_sig == GENERIC and info.epi_sig == sig, f"signature {info.epi_sig} (generic run: {info_g.epi_sig}), expected {sig}"
    assert torch.equal(out.view(torch.int32), out_g.view(torch.int32)), "fp32 output differs from the generic signature's"
    if sv:
        assert torch.equal(hm[0], hm_g[0]) and torch.equal(hm[1], hm_g[1]), "bf16 hi / mid differ from the generic signature's"
    ref, bound = c.reference(info)
    if sig & OUT:
        c.check_out(ref, bound, f"signature {sig}")
    if not sv:
        return
    hi, mid, inside = sv
    hic, midc = hm[0].cpu(), hm[1].cpu()
    assert torch.all(hic[~inside] == SENT16) and torch.all(midc[~inside] == SENT16), "out_sv: write outside the interior slice"
    sl = (slice(None), slice(1, 1 + c.Ho), slice(1, 1 + c.Wo), slice(64, 264))
    got_hi, got_mid = hic[sl].permute(0, 3, 1, 2), midc[sl].permute(0, 3, 1, 2)
    if sig & OUT:
        v = c.y().to(torch.float32)
        if sig & OS_AFFINE:
            v = v * c.os_s[None, :, None, None] + c.os_t[None, :, None, None]
            if sig & OS_RELU:
                v = v.clamp_min(0)
        want_hi, want_mid = host_split(v)
        assert torch.equal(got_hi, want_hi) and torch.equal(got_mid, want_mid), "out_sv: hi / mid differ from the split of out"
        return
    if sig & OS_AFFINE:
        s64, t64 = c.os_s.to(torch.float64)[None, :, None, None], c.os_t.to(torch.float64)[None, :, None, None]
        ref = ref * s64 + t64
        bound = bound * s64.abs() + ulp32(ref)
        if sig & OS_RELU:
            ref = ref.clamp_min(0)
    got = split_value(got_hi, got_mid)
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    assert torch.all(err <= bound + 2.0 ** -16 * ref.abs() + 1e-30), f"out_sv: error {err.max().item():.3g}"

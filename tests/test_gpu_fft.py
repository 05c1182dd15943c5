"""The inpainter's two real 2-D FFTs (LaMa's FourierUnit: torch.fft.rfftn / irfftn over (h, w), norm="ortho") against torch float64
on the CPU, never another kernel of the library, through the test hook mitb_test_fft, which launches them as lama.cu does:

* planar (fft.cu, run_ffc_layer): any 1 <= h, w <= 4096.  Stockham stages of radix 4, 2, 3, 5, 7 and a generic direct-sum stage for
  every other prime; forward = row pass (two real rows of a plane packed into one complex FFT, then separated) + column pass (scaled
  by 1/sqrt(hw)); inverse = column pass + row pass (two half-spectrum rows packed, Im of the DC / Nyquist bins dropped, scale, + the
  residual);
* NHWC (fft_nhwc.cu, run_ffc_layer_fast): {2,3,5}-smooth h, w <= 512, channel pairs packed into one complex FFT, in-place
  decimation-in-frequency stages of radix 16 (4 x 4) and 12 (4 x 3) fused in registers, 4, 2, 3 and 5; the forward emits the
  spectrum as fp32 and / or bf16 hi / mid, the inverse adds the residual and emits fp32 and / or hi / mid at a channel offset.

Error bounds (u = 2^-24, gamma_k = k u / (1 - k u)).  A multiplication by a twiddle factor read from the fp32 table (computed in
double, rounded once) or by a rounded constant costs mu = sqrt(2) gamma_2 + u relative to the product: sqrt(2) gamma_2 for the
complex product with or without a fused multiply-add, u for the rounded factor.  A complex add / sub costs u relative to its result
(each component rounded once); rot90, negation and the 0.5 factors are exact.  Each stage then costs, relative to the 2-norm of the
stage's output (the stages are unitary up to a factor sqrt(r), so a relative error passes every later stage unamplified):

  closed forms   r = 2: u + mu          r = 4: 2u + mu (two add levels)
                 r = 16 (NHWC): 4u + mu (inner twiddles w16^k) + mu       r = 12 (NHWC): 2u + mu (inner w12^k) + eta_3 + mu
  direct sums    one output is a sum of r rounded products; each term passes through D roundings (the product, its rounded
                 factor and the additions after it), so |err_k| <= 2 gamma_D sum_j |a_j| (the 2 covers both components) and,
                 with sum_j |a_j| <= sqrt(r) ||a||_2 and ||y||_2 = sqrt(r) ||a||_2, eta_r = 2 sqrt(r) gamma_D: the bound grows with
                 sqrt(r) on top of D.  Planar 3, 5, 7 and generic r: D = r + 2 (sequential accumulation), + mu for the stage
                 twiddle.  NHWC 3: D = 4, NHWC 5: D = 6 (symmetric sums), + mu.  For r = 181, eta = 2 sqrt(181) gamma_183 + mu.

eta(n) = prod_s (1 + eta_s) - 1 over the stages of the length-n plan, read from the hook's record of the plan as it was built.

Random inputs, normwise per (image, channel) plane.  Forward: the row FFT of a packed pair has error <= eta(w) ||Z||; separating the
two real rows (z_k + conj z_{w-k}) / 2 is an isometry from the full complex spectrum onto the two full real spectra and adds u; the
column FFT adds eta(h); the 1/sqrt(hw) scale is a rounded constant and a product (2u).  So
  ||y^ - y||_2 <= gamma_f ||x||_2,   gamma_f = (1 + eta(w))(1 + u)(1 + eta(h))(1 + u)^2 - 1.
Inverse: the column FFT adds eta(h); packing A + iB and its conjugate mirror adds u and doubles the energy of the interior bins (the
sqrt(2)); the row FFT adds eta(w); scale 2u; the residual add is one rounding of the result:
  ||y^ - y||_2 <= gamma_i sqrt(2) ||F||_2 + u ||y + add||_2,   gamma_i = (1 + eta(h))(1 + u)(1 + eta(w))(1 + u)^2 - 1.
The planar path packs two rows of one plane, so these hold per plane.  The NHWC path packs channels 2p and 2p + 1, whose errors mix:
there the bound holds for the pair, and each channel of the pair is checked against the pair's ||x|| (resp. ||F||).

Impulse inputs, per element.  Every intermediate value of an FFT is a partial DFT over a subset of its input, and a butterfly
combines disjoint subsets, so a stage's per-output error is at most kappa_s ||x||_1, kappa_s = 2 gamma_D + (twiddle mus), with
D = 1, 2, 4, 4 for the closed forms 2, 4, 16, 12 (add levels, the inner twiddles of 16 and 12 counted as an extra mu) and the direct
sums as above, without the sqrt(r).  kappa(n) = prod_s (1 + kappa_s) - 1.  An impulse (||x||_1 = 1, the pair partner's row zero)
gives every output magnitude 1/sqrt(hw), and
  |y^ - y| <= ((1 + kappa(w))(1 + sqrt(2) u)(1 + kappa(h))(1 + u)^2 - 1) / sqrt(hw);
a single bin F per plane (its pair partner a single bin too) gives a row input with ||X||_1 <= 2 (|F_a| + |F_b|), so
  |y^ - y| <= 2 (|F_a| + |F_b|) ((1 + kappa(h))(1 + sqrt(2) u)(1 + kappa(w))(1 + u)^2 - 1) / sqrt(hw).
No bound is fitted to observed errors; the worst error-to-bound ratio per implementation and case family is printed at the end.

Bit-exact relations: hi = bf16_rn(out) and mid = bf16_rn(out - hi) of the same call; a split-only call, a force_plain call (plain
loads where the TMA box would run), image i of an N-image call and a channel slice give the same bits as their counterparts.
Every element a call must not write holds a NaN-payload sentinel before and after the call, and input channels outside the slice
are NaN, so a read of them would show in the output.  The last test asserts from the hook's records that the cases reached every
radix (on NHWC also in a non-last stage, where its twiddle branch runs), the TMA box and the plain loads of both NHWC passes, and
full and partial planar row and column batches."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

PLANAR, NHWC = 0, 1
IMPL = {PLANAR: "planar", NHWC: "nhwc"}
SENT32 = 0x7FC0DEAD            # fp32 NaN with a payload no kernel produces
SENT16 = 0x7FDE                # bf16 NaN with a payload
TAIL = 37                      # sentinel elements past every output buffer
U = 2.0 ** -24
RECORDS = []                   # (impl, inverse, N, h, w, C, info fields) of every call
RATIOS = {}                    # (impl, family) -> worst error / bound


def gamma(k):
    return k * U / (1 - k * U)


MU = math.sqrt(2) * gamma(2) + U


def stage_eta(impl, r):
    """normwise relative error of one stage (module docstring)"""
    if r == 2:
        return U + MU
    if r == 4:
        return 2 * U + MU
    if impl == NHWC:
        eta3 = 2 * math.sqrt(3) * gamma(4)
        return {16: 4 * U + 2 * MU, 12: 2 * U + MU + eta3 + MU, 3: eta3 + MU, 5: 2 * math.sqrt(5) * gamma(6) + MU}[r]
    return 2 * math.sqrt(r) * gamma(r + 2) + MU


def stage_kappa(impl, r):
    """per-output error of one stage relative to the l1 norm of the transform's input (module docstring)"""
    if r == 2:
        return 2 * gamma(1) + MU
    if r == 4:
        return 2 * gamma(2) + MU
    if impl == NHWC:
        return {16: 2 * gamma(4) + 2 * MU, 12: 2 * gamma(2) + MU + 2 * gamma(4) + MU, 3: 2 * gamma(4) + MU, 5: 2 * gamma(6) + MU}[r]
    return 2 * gamma(r + 2) + MU


def compose(f, impl, radices):
    p = 1.0
    for r in radices:
        p *= 1 + f(impl, r)
    return p - 1


def radices(info, which):
    n = getattr(info, which + "_nst")
    return list(getattr(info, which + "_radix")[:n])


def gamma_total(impl, info, kind, sep):
    """(1 + e(first pass))(1 + sep)(1 + e(second pass))(1 + u)^2 - 1, e = eta or kappa"""
    f = stage_eta if kind == "norm" else stage_kappa
    eh, ew = compose(f, impl, radices(info, "h")), compose(f, impl, radices(info, "w"))
    return (1 + eh) * (1 + sep) * (1 + ew) * (1 + U) ** 2 - 1


def note(impl, family, ratio):
    key = (IMPL[impl], family)
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)


@pytest.fixture(scope="module")
def eng():
    import os
    from mit_b200.engine import get_engine
    torch.set_num_threads(max(1, min(64, os.cpu_count() or 1)))     # the float64 references' intra-op pool
    return get_engine("cuda:0")


# ---------------------------------------------------------------------------------------------------------------------------------
# the hook

def sentinel(n, bits=SENT32, dtype=torch.int32):
    return torch.full((n + TAIL,), bits, dtype=dtype, device="cuda")


def f32(t):
    return t.view(torch.float32)


class Result:
    pass


def run(eng, impl, inverse, N, h, w, C_, x, *, in_cs=None, in_coff=0, out=True, out_cs=None, out_coff=0, sv=None, add=None,
        add_cs=None, add_coff=0, force_plain=False):
    """One mitb_test_fft call.  x: the logical input, NHWC [N][h][W][c] or planar [N*c][h][W] (c = C or 2C, W = w or w/2+1), as a CPU
    tensor; add likewise [N][h][w][C] / [N*C][h][w].  sv = None or (C_sv, coff) of the split output.  Returns the logical outputs
    (fp32 and / or hi / mid as int16 bit patterns) after checking every sentinel."""
    from mit_b200 import _lib as L
    w2 = w // 2 + 1
    Win, Wout = (w2, w) if inverse else (w, w2)
    cin, cout = (2 * C_, C_) if inverse else (C_, 2 * C_)
    d = L.MitbTestFftDesc()
    d.impl, d.inverse, d.N, d.h, d.w, d.C, d.force_plain = impl, int(inverse), N, h, w, C_, int(force_plain)
    keep = []

    def backing(t, cs, coff, c, W):
        """the device tensor holding t at channels [coff, coff + c) of cs (NaN elsewhere)"""
        if impl == PLANAR:
            b = t.to(torch.float32).contiguous().reshape(-1).cuda()
        else:
            b = f32(torch.full((N, h, W, cs), SENT32, dtype=torch.int32))
            b[..., coff:coff + c] = t.to(torch.float32)
            b = b.reshape(-1).cuda()
        keep.append(b)
        return b

    in_cs = in_cs or cin
    xb = backing(x, in_cs, in_coff, cin, Win)
    d.__setattr__("in", L.MitbTestView(xb.data_ptr(), in_cs if impl == NHWC else 0, in_coff, 0, 0))
    ob = None
    if out:
        out_cs = out_cs or cout
        ob = f32(sentinel(N * h * Wout * out_cs if impl == NHWC else N * cout * h * Wout))
        d.out = L.MitbTestView(ob.data_ptr(), out_cs if impl == NHWC else 0, out_coff, 0, 0)
    if add is not None:
        add_cs = add_cs or C_
        ab = backing(add, add_cs, add_coff, C_, w)
        d.add = L.MitbTestView(ab.data_ptr(), add_cs if impl == NHWC else 0, add_coff, 0, 0)
    hb = mb = None
    if sv is not None:
        csv, scoff = sv
        hb, mb = sentinel(N * h * Wout * csv, SENT16, torch.int16), sentinel(N * h * Wout * csv, SENT16, torch.int16)
        d.out_sv = L.MitbTestSplit(hb.data_ptr(), mb.data_ptr(), csv, h, Wout, 0, 0, scoff)
    info = L.MitbTestFftInfo()
    eng._call(eng.lib.mitb_test_fft, C.byref(d), C.byref(info), eng._stream())
    torch.cuda.synchronize()
    RECORDS.append((impl, bool(inverse), N, h, w, C_, info.h_nst, list(info.h_radix), info.w_nst, list(info.w_radix), info.rows_tma,
                    info.rows_box_rows, info.cols_tma, info.cols_box_rows, info.P, info.CB))
    res = Result()
    res.info = info
    res.out = res.hi = res.mid = None
    if ob is not None:
        o = ob.cpu()
        n = o.numel() - TAIL
        assert torch.all(o[n:].view(torch.int32) == SENT32), "fp32 output: write past the buffer"
        o = o[:n]
        if impl == NHWC:
            o = o.view(N, h, Wout, out_cs)
            outside = torch.cat([o[..., :out_coff], o[..., out_coff + cout:]], -1)
            assert torch.all(outside.contiguous().view(torch.int32) == SENT32), "fp32 output: write outside the channel slice"
            o = o[..., out_coff:out_coff + cout]
        res.out = o.contiguous()
    if hb is not None:
        csv, scoff = sv
        for name, b in (("hi", hb), ("mid", mb)):
            t = b.cpu()
            n = t.numel() - TAIL
            assert torch.all(t[n:] == SENT16), f"{name}: write past the buffer"
            t = t[:n].view(N, h, Wout, csv)
            outside = torch.cat([t[..., :scoff], t[..., scoff + cout:]], -1)
            assert torch.all(outside == SENT16), f"{name}: write outside [sv_coff, sv_coff + C)"
            setattr(res, name, t[..., scoff:scoff + cout].contiguous())
    return res


# ---------------------------------------------------------------------------------------------------------------------------------
# layouts: everything is compared as planes [P][h][W] (P = N*C), spectra complex

def nhwc_planes(t):
    """[N][h][W][c] -> [N*c][h][W]"""
    N, h, W, c = t.shape
    return t.permute(0, 3, 1, 2).reshape(N * c, h, W)


def planes_nhwc(t, N):
    P, h, W = t.shape
    return t.reshape(N, P // N, h, W).permute(0, 2, 3, 1)


def spec_planes(o, N, C_):
    """NHWC fp32 spectrum output [N][h][w2][2C] -> complex128 [N*C][h][w2]"""
    Nn, h, w2, _ = o.shape
    o = o.to(torch.float64).view(Nn, h, w2, C_, 2).permute(0, 3, 1, 2, 4)
    return torch.complex(o[..., 0], o[..., 1]).reshape(N * C_, h, w2)


def planar_spec(o, N, C_, h, w2):
    o = o.to(torch.float64).view(N * C_, 2, h, w2)
    return torch.complex(o[:, 0], o[:, 1])


def got_spec(res, impl, N, C_, h, w2):
    if impl == NHWC:
        return spec_planes(res.out, N, C_)
    return planar_spec(res.out, N, C_, h, w2)


def got_real(res, impl, N, C_, h, w):
    if impl == NHWC:
        return nhwc_planes(res.out.to(torch.float64))
    return res.out.to(torch.float64).view(N * C_, h, w)


def spec_input(F, impl, N):
    """complex [N*C][h][w2] -> the layout the inverse reads"""
    P, h, w2 = F.shape
    if impl == NHWC:
        return torch.stack((F.real, F.imag), -1).reshape(N, P // N, h, w2, 2).permute(0, 2, 3, 1, 4).reshape(N, h, w2, 2 * (P // N)).float()
    return torch.stack((F.real, F.imag), 1).reshape(2 * P, h, w2).float()


def real_input(x, impl, N):
    """real [N*C][h][w] -> the layout the forward reads"""
    return planes_nhwc(x, N).contiguous() if impl == NHWC else x


def pair_norm(v, impl, N):
    """per plane: ||v|| of the plane (planar) or of its NHWC channel pair"""
    n = v.reshape(v.shape[0], -1).norm(dim=1)
    if impl == NHWC:
        q = n.view(N, -1)
        if q.shape[1] % 2 == 0:
            q = (q.view(N, -1, 2) ** 2).sum(-1).sqrt().repeat_interleave(2, 1)
        n = q.reshape(-1)
    return n


def check_forward(res, x64, impl, N, C_, h, w, family):
    ref = torch.fft.rfftn(x64, dim=(-2, -1), norm="ortho")
    got = got_spec(res, impl, N, C_, h, w // 2 + 1)
    err = (got - ref).reshape(N * C_, -1).abs().norm(dim=1)
    bound = gamma_total(impl, res.info, "norm", U) * pair_norm(x64, impl, N)
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    note(impl, family, ratio)
    assert torch.isfinite(got).all() and torch.all(err <= bound), f"{IMPL[impl]} rfft2 {N}x{h}x{w}x{C_} {family}: error / bound {ratio:.3g}"
    return ratio


def check_inverse(res, F64, add64, impl, N, C_, h, w, family):
    ref = torch.fft.irfftn(F64, s=(h, w), dim=(-2, -1), norm="ortho")
    if add64 is not None:
        ref = ref + add64
    got = got_real(res, impl, N, C_, h, w)
    err = (got - ref).reshape(N * C_, -1).norm(dim=1)
    bound = gamma_total(impl, res.info, "norm", U) * math.sqrt(2) * pair_norm(F64, impl, N) + U * ref.reshape(N * C_, -1).norm(dim=1)
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    note(impl, family, ratio)
    assert torch.isfinite(got).all() and torch.all(err <= bound), f"{IMPL[impl]} irfft2 {N}x{h}x{w}x{C_} {family}: error / bound {ratio:.3g}"
    return ratio


def bf16_bits(v):
    return v.to(torch.bfloat16).view(torch.int16)


def check_split(res):
    """hi = bf16_rn(out), mid = bf16_rn(out - hi), bit for bit"""
    hi = bf16_bits(res.out)
    assert torch.equal(res.hi, hi), f"hi differs from bf16_rn(out) on {(res.hi != hi).sum().item()} elements"
    rest = res.out - res.hi.view(torch.bfloat16).float()
    mid = bf16_bits(rest)
    assert torch.equal(res.mid, mid), f"mid differs from bf16_rn(out - hi) on {(res.mid != mid).sum().item()} elements"


# ---------------------------------------------------------------------------------------------------------------------------------
# every length: impulses (forward) and single bins (inverse)

def smooth(n):
    for p in (2, 3, 5):
        while n % p == 0:
            n //= p
    return n == 1


PLANAR_LENGTHS = list(range(1, 513)) + [1021, 2048, 4096]
NHWC_LENGTHS = [n for n in range(2, 513) if smooth(n)]
BIN = complex(0.75, -0.5)        # the value of every single bin (its imaginary part also on DC / Nyquist)


def impulse_case(impl, n, as_w):
    """(N, h, w, C, x [P][h][w] float64): one impulse per plane (planar) / channel (NHWC) at every position of the length-n axis;
    NHWC channel pairs put their two impulses into different rows"""
    small = 1 if impl == PLANAR else 2
    h, w = (small, n) if as_w else (n, small)
    P = n if impl == PLANAR else n + (n & 1)
    x = torch.zeros(P, h, w, dtype=torch.float64)
    p = torch.arange(P)
    pos = p % n
    if impl == NHWC:
        other = p % 2                                   # pair (2q, 2q + 1): rows 0 / 1 (as w) or columns 0 / 1 (as h)
    else:
        other = p % small
    ys, xs = (other, pos) if as_w else (pos, other)
    if impl == NHWC and not as_w:
        ys = pos                                        # rows differ: pos of 2q and 2q + 1 differ (n >= 2)
    x[p, ys, xs] = 1.0
    return 1, h, w, P, x


def bin_case(impl, n, as_w):
    """(N, h, w, C, F [P][h][w2] complex128): one bin per plane / channel, every bin position of the length-n axis"""
    small = 1 if impl == PLANAR else 2                  # NHWC: a Nyquist column when n runs along h
    h, w = (small, n) if as_w else (n, small)
    w2 = w // 2 + 1
    m = w2 if as_w else h
    P = m if impl == PLANAR else m + (m & 1)
    F = torch.zeros(P, h, w2, dtype=torch.complex128)
    p = torch.arange(P)
    pos = p % m
    other = p % (h if as_w else w2)
    ky, kx = (other, pos) if as_w else (pos, other)
    F[p, ky, kx] = BIN
    return 1, h, w, P, F


def check_impulses(eng, impl, n, as_w):
    N, h, w, P, x = impulse_case(impl, n, as_w)
    res = run(eng, impl, False, N, h, w, P, real_input(x.float(), impl, N))
    ref = torch.fft.rfftn(x, dim=(-2, -1), norm="ortho")
    got = got_spec(res, impl, N, P, h, w // 2 + 1)
    err = (got - ref).abs()
    bound = gamma_total(impl, res.info, "elem", math.sqrt(2) * U) / math.sqrt(h * w)
    ratio = err.max().item() / bound            # NaN (an unwritten or poisoned element) fails the test below
    note(impl, "impulse", ratio)
    assert ratio <= 1, f"{IMPL[impl]} rfft2 impulses {h}x{w}: error / bound {ratio:.3g}"

    N, h, w, P, F = bin_case(impl, n, as_w)
    res = run(eng, impl, True, N, h, w, P, spec_input(F, impl, N))
    ref = torch.fft.irfftn(F, s=(h, w), dim=(-2, -1), norm="ortho")
    got = got_real(res, impl, N, P, h, w)
    err = (got - ref).abs()
    bound = 4 * abs(BIN) * gamma_total(impl, res.info, "elem", math.sqrt(2) * U) / math.sqrt(h * w)
    ratio = err.max().item() / bound
    note(impl, "single bin", ratio)
    assert ratio <= 1, f"{IMPL[impl]} irfft2 single bins {h}x{w}: error / bound {ratio:.3g}"


@pytest.mark.parametrize("as_w", [True, False], ids=["w", "h"])
def test_planar_every_length(eng, as_w):
    """planar: every n from 1 to 512, 1021, 2048 and 4096, as w (h = 1) and as h (w = 1)"""
    for n in PLANAR_LENGTHS:
        check_impulses(eng, PLANAR, n, as_w)


@pytest.mark.parametrize("as_w", [True, False], ids=["w", "h"])
def test_nhwc_every_length(eng, as_w):
    """NHWC: all 67 {2,3,5}-smooth n from 2 to 512, as w and as h; C = n (rounded up to even) takes both load paths"""
    assert len(NHWC_LENGTHS) == 67
    for n in NHWC_LENGTHS:
        check_impulses(eng, NHWC, n, as_w)


# ---------------------------------------------------------------------------------------------------------------------------------
# production shapes, random data

def rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64) * scale


def rand_spec(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.complex(torch.randn(*shape, generator=g, dtype=torch.float64), torch.randn(*shape, generator=g, dtype=torch.float64))


def round32(t):
    """t rounded to the fp32 (complex64) values the kernels receive"""
    return (t.to(torch.complex64) if t.is_complex() else t.float()).to(t.dtype)


@pytest.mark.parametrize("h,w", [(256, 192), (320, 240)])
def test_nhwc_production(eng, h, w):
    """run_ffc_layer_fast's calls: C = 192, fp32 and split outputs in one call, the inverse with the residual; split-only and
    force_plain calls give the same bits, and image i of the two-image call equals a one-image call on image i"""
    C_, N = 192, 2
    seed = h * 1000 + w + N
    x = round32(rand((N * C_, h, w), seed))
    xin = real_input(x.float(), NHWC, N)
    fw = run(eng, NHWC, False, N, h, w, C_, xin, sv=(2 * C_, 0))
    assert fw.info.rows_tma == 1 and fw.info.cols_tma == 1
    check_forward(fw, x, NHWC, N, C_, h, w, "production")
    check_split(fw)
    only = run(eng, NHWC, False, N, h, w, C_, xin, out=False, sv=(2 * C_, 0))
    assert torch.equal(only.hi, fw.hi) and torch.equal(only.mid, fw.mid)
    plain = run(eng, NHWC, False, N, h, w, C_, xin, sv=(2 * C_, 0), force_plain=True)
    assert plain.info.rows_tma == 0 and plain.info.cols_tma == 0
    assert torch.equal(plain.out.view(torch.int32), fw.out.view(torch.int32)) and torch.equal(plain.hi, fw.hi)

    F = round32(rand_spec((N * C_, h, w // 2 + 1), seed + 1))       # non-Hermitian, like the spectrum after conv + ReLU
    add = round32(rand((N * C_, h, w), seed + 2))
    Fin, addin = spec_input(F, NHWC, N), real_input(add.float(), NHWC, N)
    iv = run(eng, NHWC, True, N, h, w, C_, Fin, add=addin, sv=(C_, 0))
    assert iv.info.cols_tma == 1 and iv.info.rows_tma == 0
    check_inverse(iv, F, add, NHWC, N, C_, h, w, "production")
    check_split(iv)
    only = run(eng, NHWC, True, N, h, w, C_, Fin, out=False, add=addin, sv=(C_, 0))
    assert torch.equal(only.hi, iv.hi) and torch.equal(only.mid, iv.mid)
    plain = run(eng, NHWC, True, N, h, w, C_, Fin, add=addin, sv=(C_, 0), force_plain=True)
    assert plain.info.cols_tma == 0
    assert torch.equal(plain.out.view(torch.int32), iv.out.view(torch.int32)) and torch.equal(plain.hi, iv.hi)
    for i in range(N):
        one = run(eng, NHWC, False, 1, h, w, C_, xin[i:i + 1].contiguous(), sv=(2 * C_, 0))
        assert torch.equal(one.out.view(torch.int32), fw.out[i:i + 1].view(torch.int32)) and torch.equal(one.hi, fw.hi[i:i + 1])
        one = run(eng, NHWC, True, 1, h, w, C_, Fin[i:i + 1].contiguous(), add=addin[i:i + 1].contiguous(), sv=(C_, 0))
        assert torch.equal(one.out.view(torch.int32), iv.out[i:i + 1].view(torch.int32)) and torch.equal(one.mid, iv.mid[i:i + 1])


@pytest.mark.parametrize("h,w,N", [(181, 256, 2), (256, 181, 1), (182, 256, 1), (171, 256, 1)])
def test_planar_production(eng, h, w, N):
    """run_ffc_layer's calls: N * 192 planes, the inverse with the residual (odd and even h and w, partial row and column batches);
    image i of a two-image call equals a one-image call on image i"""
    C_ = 192
    seed = h * 1000 + w + 7 * N
    x = round32(rand((N * C_, h, w), seed))
    fw = run(eng, PLANAR, False, N, h, w, C_, x.float())
    check_forward(fw, x, PLANAR, N, C_, h, w, "production")
    F = round32(rand_spec((N * C_, h, w // 2 + 1), seed + 1))
    add = round32(rand((N * C_, h, w), seed + 2))
    iv = run(eng, PLANAR, True, N, h, w, C_, spec_input(F, PLANAR, N), add=add.float())
    check_inverse(iv, F, add, PLANAR, N, C_, h, w, "production")
    for i in range(N if N > 1 else 0):
        one = run(eng, PLANAR, False, 1, h, w, C_, x[i * C_:(i + 1) * C_].float())
        assert torch.equal(one.out.view(torch.int32), fw.out.view(N, -1)[i].view(torch.int32))
        one = run(eng, PLANAR, True, 1, h, w, C_, spec_input(F[i * C_:(i + 1) * C_], PLANAR, 1), add=add[i * C_:(i + 1) * C_].float())
        assert torch.equal(one.out.view(torch.int32), iv.out.view(N, -1)[i].view(torch.int32))


SMALL_PLANAR = [(8, 8, 6), (16, 12, 6), (20, 14, 6), (11, 15, 6), (32, 24, 6), (256, 192, 3), (40, 30, 6), (97, 6, 6), (6, 97, 6),
                (13, 128, 6), (24, 20, 2)]
SMALL_NHWC = [(1, 16, 12, 64), (2, 8, 8, 2), (1, 20, 30, 6), (1, 256, 192, 64), (1, 320, 240, 64), (2, 32, 24, 192), (1, 5, 9, 70),
              (1, 64, 50, 34)]


@pytest.mark.parametrize("case", [(PLANAR, 1) + c[:2] + c[2:] for c in SMALL_PLANAR] + [(NHWC,) + c[:1] + c[1:] for c in SMALL_NHWC],
                         ids=lambda c: f"{IMPL[c[0]]}-{c[1]}x{c[2]}x{c[3]}x{c[4]}")
def test_random_small(eng, case):
    """small and odd shapes, random data, both directions, the inverse with and without the residual"""
    impl, N, h, w, C_ = case
    seed = impl * 7 + N * 11 + h * 1000 + w + C_
    x = round32(rand((N * C_, h, w), seed))
    check_forward(run(eng, impl, False, N, h, w, C_, real_input(x.float(), impl, N)), x, impl, N, C_, h, w, "random small")
    F = round32(rand_spec((N * C_, h, w // 2 + 1), seed + 1))
    add = round32(rand((N * C_, h, w), seed + 2))
    Fin = spec_input(F, impl, N)
    check_inverse(run(eng, impl, True, N, h, w, C_, Fin), F, None, impl, N, C_, h, w, "random small")
    check_inverse(run(eng, impl, True, N, h, w, C_, Fin, add=real_input(add.float(), impl, N)), F, add, impl, N, C_, h, w, "random small")


# ---------------------------------------------------------------------------------------------------------------------------------
# views and edges (NHWC)

@pytest.mark.parametrize("C_", [2, 34, 96, 128])
@pytest.mark.parametrize("h,w", [(24, 20), (45, 32)])
def test_nhwc_views(eng, h, w, C_):
    """input, residual and output channel slices (cs > C, coff != 0), the split output at sv_coff 0 and inside a wider split tensor;
    C = 2 and C = 34 take the plain loads, 96 the TMA box in the column passes only, 128 in every pass that has one.  A slice gives
    the bits of the dense view."""
    N = 2
    seed = h * 100 + w + C_
    x = round32(rand((N * C_, h, w), seed))
    xin = real_input(x.float(), NHWC, N)
    dense = run(eng, NHWC, False, N, h, w, C_, xin, sv=(2 * C_, 0))
    check_forward(dense, x, NHWC, N, C_, h, w, "views")
    check_split(dense)
    sl = run(eng, NHWC, False, N, h, w, C_, xin, in_cs=C_ + 72, in_coff=68, sv=(2 * C_, 0))
    assert torch.equal(sl.out.view(torch.int32), dense.out.view(torch.int32)) and torch.equal(sl.hi, dense.hi) and torch.equal(sl.mid, dense.mid)

    F = round32(rand_spec((N * C_, h, w // 2 + 1), seed + 1))
    add = round32(rand((N * C_, h, w), seed + 2))
    Fin, addin = spec_input(F, NHWC, N), real_input(add.float(), NHWC, N)
    dense = run(eng, NHWC, True, N, h, w, C_, Fin, add=addin, sv=(C_, 0))
    check_inverse(dense, F, add, NHWC, N, C_, h, w, "views")
    check_split(dense)
    for sv in ((C_ + 64, 32), (C_ + 2, 2)):
        sl = run(eng, NHWC, True, N, h, w, C_, Fin, in_cs=2 * C_ + 8, in_coff=4, add=addin, add_cs=C_ + 10, add_coff=6,
                 out_cs=C_ + 4, out_coff=2, sv=sv)
        assert torch.equal(sl.out.view(torch.int32), dense.out.view(torch.int32)), sv
        assert torch.equal(sl.hi, dense.hi) and torch.equal(sl.mid, dense.mid), sv
        only = run(eng, NHWC, True, N, h, w, C_, Fin, in_cs=2 * C_ + 8, in_coff=4, add=addin, add_cs=C_ + 10, add_coff=6, out=False, sv=sv)
        assert torch.equal(only.hi, dense.hi) and torch.equal(only.mid, dense.mid), sv


def test_public_fft_entry_points(eng):
    """mitb_op_rfft2 / irfft2 / rfft2_nhwc / irfft2_nhwc (the C ABI) run the same kernels as the hook: same bits"""
    g = torch.Generator().manual_seed(3)
    c, h, w = 6, 20, 14
    x = torch.randn(c, h, w, generator=g)
    spec = eng.rfft2(x).cpu()
    assert torch.equal(spec.reshape(-1), run(eng, PLANAR, False, 1, h, w, c, x).out.reshape(-1))
    s = torch.randn(2 * c, h, w // 2 + 1, generator=g)
    assert torch.equal(eng.irfft2(s, w).cpu().reshape(-1), run(eng, PLANAR, True, 1, h, w, c, s).out.reshape(-1))
    n, c, w = 2, 70, 30
    x = torch.randn(n, h, w, c, generator=g)
    assert torch.equal(eng.rfft2_nhwc(x).cpu(), run(eng, NHWC, False, n, h, w, c, x).out)
    s = torch.randn(n, h, w // 2 + 1, 2 * c, generator=g)
    add = torch.randn(n, h, w, c, generator=g)
    assert torch.equal(eng.irfft2_nhwc(s, w, add).cpu(), run(eng, NHWC, True, n, h, w, c, s, add=add).out)
    assert torch.equal(eng.irfft2_nhwc(s, w).cpu(), run(eng, NHWC, True, n, h, w, c, s).out)


# ---------------------------------------------------------------------------------------------------------------------------------

def test_zz_reachability():
    """The module's calls reached every radix of both implementations (NHWC ones also in a non-last stage), the TMA box and the
    plain loads of both NHWC passes, and full and partial planar row and column batches.  Prints the worst error-to-bound ratios."""
    if not any(r[0] == PLANAR for r in RECORDS) or not any(r[0] == NHWC for r in RECORDS) or len(RECORDS) < 1000:
        pytest.skip("only part of the module ran")
    for (impl, fam), ratio in sorted(RATIOS.items()):
        print(f"worst error / bound: {impl:6s} {fam:12s} {ratio:.3g}")
    planar_r, nhwc_any, nhwc_inner = set(), set(), set()
    tma = set()
    batches = set()
    for impl, inv, N, h, w, C_, hn, hr, wn, wr, rt, rb, ct, cb, P, CB in RECORDS:
        for n, rs in ((hn, hr), (wn, wr)):
            rs = rs[:n]
            if impl == PLANAR:
                planar_r |= {r if r <= 7 else "generic" for r in rs}
            else:
                nhwc_any |= set(rs)
                nhwc_inner |= set(rs[:-1])
        if impl == NHWC:
            tma |= {("rows", rt), ("cols", ct)}
        else:
            npairs, w2 = (h + 1) // 2, w // 2 + 1
            batches |= {("P", npairs % P == 0), ("CB", w2 % CB == 0)}
    assert planar_r == {4, 2, 3, 5, 7, "generic"}, planar_r
    assert any(r[0] == PLANAR and max(r[7][:r[6]] + r[9][:r[8]] + [0]) >= 11 for r in RECORDS)
    assert nhwc_any == {16, 12, 4, 2, 3, 5} and nhwc_inner == {16, 12, 4, 2, 3, 5}, (nhwc_any, nhwc_inner)
    assert tma == {("rows", 0), ("rows", 1), ("cols", 0), ("cols", 1)}, tma
    assert batches == {("P", True), ("P", False), ("CB", True), ("CB", False)}, batches

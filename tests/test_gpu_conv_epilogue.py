"""The fused conv epilogue contract (ConvOp in csrc/mitb_internal.h), kernel path by kernel path, through the test hook
mitb_test_conv:

    v = acc (+ add0) ; v = v*scale + shift ; v = act(v) ; v *= mul1 ; v += add1  -> fp32 out and / or bf16 hi / mid operands

The reference is torch float64 on the CPU (exact-erf GELU), never another kernel of the library.  The error bound is per element:
A = conv(|x|, |w|) in float64 is the accumulation magnitude, c*A the accumulator's error (tensor cores, bf16x3 split: c = 2^-15;
SIMT fp32: c = (K + 2) * 2^-24, the extra 2 for the rounded input prologue).  That error is carried through the chain: each fp32
operation adds one ulp of its result, multiplications scale it by |scale| / |mul1|, the activation by its Lipschitz constant plus
4 ulp of its value (GELU: plus 2^-22 |v| for the cancellation in 1 + erf, and 2e-7 |v| more for the TMA kernel's gelu_fast).
The output must satisfy |y - ref| <= that + 4 ulp(|ref|).  The per-operation ulp terms are what the fp32 epilogue itself may
round; they matter only where a residual cancels the product.

Every call fills the output buffers with a NaN sentinel first: afterwards every element inside the written slice / grid is finite
and within the bound, and every element outside it (other channels of a shared cs, off-phase pixels, the out_sv halo and other
slices) still holds the sentinel.  Where exactness is defined (out_sv next to out, in_sv against the internal split, need_px,
the split-reuse cache) the check is bit for bit.  The last test asserts that the cases together reached every kernel and every
conv_tma_kernel instantiation, so a shape change that moves a case to another path does not go unnoticed."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

NONE, RELU, GELU, SILU, SIGMOID, SIGMOID2, CLAMP01 = range(7)
KERNELS = {1: "simt", 2: "fewout", 3: "thin", 4: "gather", 5: "gather_splitk", 6: "tma", 7: "stem8"}
PATHS = {"auto": 0, "simt": 1, "gather": 2, "tma": 3}
LIPSCHITZ = [1.0, 1.0, 1.13, 1.1, 0.25, 0.0625, 1.0]
SENT32 = 0x7FC0DEAD            # fp32 NaN with a payload no kernel produces
SENT16 = 0x7FDD                # bf16 NaN
TRACES = []                    # (kernel, bn, vec2, tma_act, splits) of every hook call of this module
RAN = set()


@pytest.fixture(scope="module")
def eng():
    from mit_b200.engine import get_engine
    e = get_engine("cuda:0")
    yield e
    e.set_tensor_cores(True)


def _lib():
    from mit_b200 import _lib as L
    return L


def act64(v, act):
    if act == RELU:
        return v.clamp_min(0)
    if act == GELU:
        return 0.5 * v * (1 + torch.erf(v / 2 ** 0.5))
    if act == SILU:
        return v * torch.sigmoid(v)
    if act == SIGMOID:
        return torch.sigmoid(v)
    if act == SIGMOID2:
        return torch.sigmoid(torch.sigmoid(v))
    if act == CLAMP01:
        return v.clamp(0, 1)
    return v


def ulp32(v):
    _, e = torch.frexp(v.abs().to(torch.float64))
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 24)


def conv64(x, w, stride, pad_y, pad_x, mode):
    if mode == 1 and (pad_y or pad_x):
        return F.conv2d(F.pad(x, (pad_x, pad_x, pad_y, pad_y), mode="reflect"), w, stride=stride)
    return F.conv2d(x, w, stride=stride, padding=(pad_y, pad_x))


def host_split(v):
    """bf16 hi / mid of fp32 values, both round-to-nearest-even: the split every kernel of the library makes."""
    v = v.to(torch.float32)
    hi = v.to(torch.bfloat16)
    mid = (v - hi.to(torch.float32)).to(torch.bfloat16)
    return hi.view(torch.int16), mid.view(torch.int16)


def split_value(hi, mid):
    return hi.view(torch.bfloat16).to(torch.float64) + mid.view(torch.bfloat16).to(torch.float64)


def sel(buf, planar, coff, C, phase, Ho, Wo):
    """the logical [N, C, Ho, Wo] slice of an NHWC [N, H, W, cs] or planar [N, cs, H, W] backing tensor"""
    oym, oya, oxm, oxa = phase
    if planar:
        return buf[:, coff:coff + C, oya::oym, oxa::oxm][:, :, :Ho, :Wo]
    return buf[:, oya::oym, oxa::oxm, coff:coff + C][:, :Ho, :Wo].permute(0, 3, 1, 2)


def sentinel_f32(shape):
    return torch.full(shape, SENT32, dtype=torch.int32, device="cuda").view(torch.float32)


def launch(eng, d):
    L = _lib()
    info = L.MitbTestConvInfo()
    eng._call(eng.lib.mitb_test_conv, C.byref(d), C.byref(info), eng._stream())
    TRACES.append((KERNELS.get(info.kernel, "?"), info.bn, info.vec2, info.tma_act, info.splits))
    return info


def spec(**kw):
    s = dict(n=1, cin=64, h=12, w=20, cout=200, k=3, stride=1, pad=None, mode=0, act=NONE, path="tma", bn=0, shift=True, scale=False,
             mul1=False, add0=None, add1=None, add1_out=False, in_pro=False, in_cs=None, in_coff=0, in_planar=False, wt_cin=None,
             out_cs=None, out_coff=0, out_planar=False, grid2=False, scale4=False, expect="tma", vec2=None, splits=None)
    s.update(kw)
    if s["pad"] is None:
        s["pad"] = s["k"] // 2
    s["in_cs"] = s["in_cs"] or s["cin"] + s["in_coff"]
    s["out_cs"] = s["out_cs"] or s["cout"] + s["out_coff"]
    s["wt_cin"] = s["wt_cin"] or s["cin"]
    return s


class Conv:
    """Device tensors + descriptor of one case, and its float64 reference."""

    def __init__(self, s, seed):
        L = _lib()
        self.s = s
        g = torch.Generator().manual_seed(seed)
        n, cin, h, w, cout, k, st, pad = s["n"], s["cin"], s["h"], s["w"], s["cout"], s["k"], s["stride"], s["pad"]
        self.Ho, self.Wo = (h + 2 * pad - k) // st + 1, (w + 2 * pad - k) // st + 1
        Ho, Wo = self.Ho, self.Wo
        self.phase = (2, 1, 2, 0) if s["grid2"] else (1, 0, 1, 0)
        oH, oW = (2 * Ho, 2 * Wo) if s["grid2"] else (Ho, Wo)
        self.oH, self.oW = oH, oW
        d = self.d = L.MitbTestConvDesc()
        self.keep = []
        # input
        xb = torch.randn((n, s["in_cs"], h, w) if s["in_planar"] else (n, h, w, s["in_cs"]), generator=g)
        self.xb = xb.cuda()
        self.keep.append(self.xb)
        xl = xb[:, s["in_coff"]:s["in_coff"] + cin] if s["in_planar"] else xb[..., s["in_coff"]:s["in_coff"] + cin].permute(0, 3, 1, 2)
        self.x64 = xl.to(torch.float64)
        d.x = self.xb.data_ptr()
        d.N, d.H, d.W, d.C, d.cs, d.coff, d.planar = n, h, w, cin, s["in_cs"], s["in_coff"], int(s["in_planar"])
        self.in_scale = self.in_shift = None
        if s["in_pro"]:
            self.in_scale, self.in_shift = torch.rand(cin, generator=g) + 0.5, torch.randn(cin, generator=g) * 0.5
            d.in_scale, d.in_shift, d.in_relu = self.dev(self.in_scale), self.dev(self.in_shift), 1
        # weights
        self.wt = torch.randn(cout, s["wt_cin"], k, k, generator=g) / (s["wt_cin"] * k * k) ** 0.5
        d.wt = self.dev(self.wt)
        d.cout, d.wt_cin, d.kh, d.kw, d.stride, d.pad_y, d.pad_x, d.pad_mode = cout, s["wt_cin"], k, k, st, pad, pad, s["mode"]
        # epilogue vectors (scale4: 4-byte but not 8-byte aligned, which keeps the tensor-core epilogue off its float2 branch)
        self.scale = (torch.rand(cout, generator=g) + 0.5) * torch.sign(torch.randn(cout, generator=g)) if s["scale"] else None
        self.shift = torch.randn(cout, generator=g) if s["shift"] else None
        self.mul1 = torch.randn(cout, generator=g) if s["mul1"] else None
        if self.scale is not None:
            d.scale = self.dev(self.scale, off4=s["scale4"])
        if self.shift is not None:
            d.shift = self.dev(self.shift)
        if self.mul1 is not None:
            d.mul1 = self.dev(self.mul1)
        d.act, d.runs = s["act"], 1
        # output, sentinel everywhere
        oshape = (n, s["out_cs"], oH, oW) if s["out_planar"] else (n, oH, oW, s["out_cs"])
        self.out = sentinel_f32(oshape)
        d.out = self.out.data_ptr()
        d.out_H, d.out_W, d.out_cs, d.out_coff, d.out_planar = oH, oW, s["out_cs"], s["out_coff"], int(s["out_planar"])
        d.oy_mul, d.oy_add, d.ox_mul, d.ox_add = self.phase
        self.written = torch.zeros(oshape, dtype=torch.bool)
        sel(self.written, s["out_planar"], s["out_coff"], cout, self.phase, Ho, Wo).fill_(True)
        # residuals
        self.res = {}
        for name in ("add0", "add1"):
            r = s[name]
            if name == "add1" and s["add1_out"]:              # in place: add1 is the output tensor itself (ocr.cu's residual)
                vals = torch.randn(n, cout, Ho, Wo, generator=g)
                host = self.out.cpu()
                sel(host, s["out_planar"], s["out_coff"], cout, self.phase, Ho, Wo).copy_(vals)
                self.out.copy_(host)
                self.res[name] = vals.to(torch.float64)
                v = getattr(d, name)
                v.p, v.cs, v.coff, v.planar = d.out, s["out_cs"], s["out_coff"], int(s["out_planar"])
                continue
            if not r:
                continue
            r = dict(cs=cout, coff=0, planar=False) if r is True else dict(dict(cs=cout, coff=0, planar=False), **r)
            b = torch.randn((n, r["cs"], oH, oW) if r["planar"] else (n, oH, oW, r["cs"]), generator=g)
            self.res[name] = sel(b, r["planar"], r["coff"], cout, self.phase, Ho, Wo).to(torch.float64)
            v = getattr(d, name)
            v.p, v.cs, v.coff, v.planar = self.dev(b), r["cs"], r["coff"], int(r["planar"])
        d.path, d.force_bn = PATHS[s["path"]], s["bn"]

    def dev(self, t, off4=False):
        if off4:
            b = torch.zeros(t.numel() + 1, device="cuda")
            b[1:].copy_(t.reshape(-1))
            self.keep.append(b)
            return b.data_ptr() + 4
        t = t.contiguous().cuda()
        self.keep.append(t)
        return t.data_ptr()

    def x_eff(self):
        x = self.x64
        if self.in_scale is not None:
            x = (x * self.in_scale.to(torch.float64)[None, :, None, None] + self.in_shift.to(torch.float64)[None, :, None, None]).clamp_min(0)
        return x[:, :self.s["wt_cin"]]

    def acc64(self):
        """(accumulator, accumulation magnitude A, K) in float64"""
        s = self.s
        x, w = self.x_eff(), self.wt.to(torch.float64)
        acc = conv64(x, w, s["stride"], s["pad"], s["pad"], s["mode"])
        A = conv64(x.abs(), w.abs(), s["stride"], s["pad"], s["pad"], s["mode"])
        return acc, A, s["k"] * s["k"] * s["cin"]

    def reference(self, info, acc=None, A=None, K=None):
        """float64 result of the chain and its per-element error bound for the kernel that ran"""
        if acc is None:
            acc, A, K = self.acc64()
        s, kern = self.s, KERNELS[info.kernel]
        tc = kern in ("gather", "gather_splitk", "tma", "stem8")
        E = A * (2.0 ** -15 if tc else (K + 2) * 2.0 ** -24)
        ch = lambda t: None if t is None else t.to(torch.float64)[None, :, None, None]
        v = acc
        if "add0" in self.res:
            v = v + self.res["add0"]
            E = E + ulp32(v)
        if self.scale is not None:
            v = v * ch(self.scale)
            E = E * ch(self.scale).abs() + ulp32(v)
        if self.shift is not None:
            v = v + ch(self.shift)
            E = E + ulp32(v)
        a = act64(v, s["act"])
        E = E * LIPSCHITZ[s["act"]] + 4 * ulp32(a)
        if s["act"] == GELU:
            E = E + v.abs() * (2.0 ** -22 + (2e-7 if info.tma_act == GELU else 0.0))
        v = a
        if self.mul1 is not None:
            v = v * ch(self.mul1)
            E = E * ch(self.mul1).abs() + ulp32(v)
        if "add1" in self.res:
            v = v + self.res["add1"]
            E = E + ulp32(v)
        return v, E + 4 * ulp32(v)

    def y(self):
        s = self.s
        return sel(self.out.cpu(), s["out_planar"], s["out_coff"], s["cout"], self.phase, self.Ho, self.Wo).to(torch.float64)

    def check_out(self, ref, bound, what=""):
        out = self.out.cpu()
        bits = out.view(torch.int32)
        assert torch.all(bits[~self.written] == SENT32), f"{what}: write outside the output slice / grid"
        y = self.y()
        assert torch.isfinite(y).all(), f"{what}: unwritten or non-finite element inside the output slice"
        err = (y - ref).abs()
        r = err / bound
        worst = r.max().item()
        at = tuple(int(i) for i in torch.unravel_index(r.argmax(), r.shape))
        assert worst <= 1.0, f"{what}: error {err[at].item():.3g} is {worst:.2f}x the bound at (n, c, y, x) = {at}"
        return worst


def expect_path(s, info):
    k = KERNELS[info.kernel]
    assert k == s["expect"], f"ran on {k}, expected {s['expect']}"
    if s["bn"]:
        assert info.bn == s["bn"]
    if s["vec2"] is not None:
        assert info.vec2 == s["vec2"], f"vec2 = {info.vec2}, expected {s['vec2']}"
    if s["splits"] is not None:
        assert (info.splits > 1) == s["splits"], f"splits = {info.splits}"


def run_case(eng, s, seed):
    c = Conv(s, seed)
    info = launch(eng, c.d)
    expect_path(s, info)
    ref, bound = c.reference(info)
    c.check_out(ref, bound, str(info.kernel))
    RAN.add(seed)
    return c, info


# ---------------------------------------------------------------------------------------------------------------------------------
# TMA-fed kernel: every activation instantiation x every N tile, each with the float2 and the scalar epilogue branch.  Cout 200 / 201
# admit every BN (and none of them divides it: every case has an N tail); M = 240 is two 128-row tiles with a ragged second one
# (k = 1: flattened rows; k = 3: 32 x 4 patches with columns 20..31 outside the image).
FEATURES = [dict(scale=True, mul1=True, add0=True, add1=True), dict(scale=True), dict(add0=True), dict(add1=True), dict(mul1=True)]
SCALAR_TRIGGERS = [dict(cout=201), dict(out_cs=203, out_coff=3), dict(add0=dict(planar=True), add1=dict(planar=True)),
                   dict(scale=True, scale4=True)]
TMA_CASES = []
for ia, act in enumerate((NONE, RELU, GELU, SILU, SIGMOID, SIGMOID2, CLAMP01)):
    for ib, bn in enumerate((32, 64, 96, 128)):
        for vec2 in (1, 0):
            i = len(TMA_CASES)
            kw = dict(FEATURES[i % 5], act=act, bn=bn, k=1 if (ia + ib) % 2 else 3, vec2=vec2)
            if not vec2:
                trig = dict(SCALAR_TRIGGERS[(ia + ib) % 4])
                if "add0" in trig:                        # planar residuals: keep the case's own residual choice, but planar
                    trig = {k: v for k, v in trig.items() if kw.get(k)} or dict(add1=dict(planar=True))
                kw.update(trig)
            TMA_CASES.append(kw)


@pytest.mark.parametrize("i", range(len(TMA_CASES)))
def test_tma_epilogue(eng, i):
    run_case(eng, spec(**TMA_CASES[i]), 1000 + i)


# ---------------------------------------------------------------------------------------------------------------------------------
# register-gather wgmma kernel (tensor cores on, TMA-fed kernel off), without and with split-K (Cin 128 3x3: 18 K blocks over 4 tiles)
ALL = dict(scale=True, mul1=True, add0=True, add1=True)
GATHER_CASES = [
    dict(ALL, act=GELU, vec2=1),
    dict(ALL, act=SIGMOID2, out_planar=True, vec2=0),
    dict(scale=True, add1_out=True, act=RELU, vec2=1),
    dict(scale=True, mul1=True, add1_out=True, out_planar=True, act=CLAMP01, vec2=0),
    dict(add0=dict(planar=True), add1=dict(cs=210, coff=6), out_cs=203, out_coff=3, act=SILU, vec2=0),
    dict(ALL, grid2=True, act=SIGMOID, vec2=1),
    dict(ALL, cin=40, act=NONE, vec2=1),                                     # Cin 40: K blocks straddle taps
    dict(ALL, k=1, in_planar=True, cin=64, act=RELU, out_planar=True, vec2=0),  # planar input (1x1)
    dict(ALL, in_pro=True, act=GELU, vec2=1),
]
for c in GATHER_CASES:
    c.setdefault("path", "gather"), c.setdefault("expect", "gather"), c.setdefault("splits", False)
GATHER_CASES += [dict(c, cin=128, h=10, w=20, expect="gather_splitk", splits=True, vec2=None) for c in GATHER_CASES[:6]]


@pytest.mark.parametrize("i", range(len(GATHER_CASES)))
def test_gather_epilogue(eng, i):
    run_case(eng, spec(**GATHER_CASES[i]), 2000 + i)


# ---------------------------------------------------------------------------------------------------------------------------------
# exact-fp32 SIMT kernel (tensor cores off): BN 128 (Cout 200) and 64 (Cout 40), NHWC and planar input; fewout (Cout <= 4)
SIMT_CASES = []
for cout, bn in ((200, 128), (40, 64)):
    for planar in (False, True):
        base = dict(cout=cout, cin=32, path="simt", expect="simt", in_planar=planar, k=1 if planar else 3)
        SIMT_CASES += [
            dict(base, **ALL, act=GELU),
            dict(base, add0=dict(planar=True), add1=dict(planar=True), out_planar=True, scale=True, act=SIGMOID2),
            dict(base, add1_out=True, mul1=True, act=RELU),
            dict(base, add1_out=True, out_planar=True, scale=True, act=SILU),
            dict(base, out_cs=cout + 7, out_coff=3, add0=dict(cs=cout + 2, coff=1), act=CLAMP01, scale=True),   # scalar stores / loads
            dict(base, **ALL, grid2=True, act=SIGMOID),
            dict(base, in_pro=True, mul1=True, act=NONE),
        ]
FEWOUT = dict(cin=16, path="simt", expect="fewout")
SIMT_CASES += [
    dict(FEWOUT, cout=3, act=CLAMP01, scale=True, mul1=True, add1=True),                 # the OCR colour head's activation
    dict(FEWOUT, cout=4, act=CLAMP01, add0=dict(planar=True), out_planar=True),
    dict(FEWOUT, cout=1, act=SIGMOID, add1_out=True, out_cs=3, out_coff=2, in_pro=True),
    dict(FEWOUT, cout=2, act=SIGMOID2, grid2=True, add0=True, scale=True),
]


@pytest.mark.parametrize("i", range(len(SIMT_CASES)))
def test_simt_epilogue(eng, i):
    run_case(eng, spec(**SIMT_CASES[i]), 3000 + i)


# ---------------------------------------------------------------------------------------------------------------------------------
# conv7_thin (7x7, Cout <= 4: shift + activation only) and the Cin = 4 stem mode of the TMA kernel (RGB padded to 4 channels; the
# 4th input channel holds noise that its zero weights must cancel)
THIN_CASES = [dict(k=7, cin=16, h=20, w=70, cout=3, act=a, path="auto", expect="thin", mode=m, out_planar=p, out_cs=cs)
              for a, m, p, cs in ((NONE, 0, False, None), (RELU, 1, True, None), (SILU, 1, False, 5), (SIGMOID, 0, True, 4))]
STEM_CASES = [dict(k=7, cin=4, wt_cin=3, cout=64, stride=st, mode=m, h=h, w=w, expect="stem8", **f)
              for st, m, h, w, f in ((1, 0, 16, 20, dict(act=RELU)), (1, 1, 16, 20, ALL), (2, 0, 24, 24, dict(scale=True, act=GELU)),
                                     (2, 1, 26, 30, dict(add1=True, mul1=True, act=SIGMOID)))]


@pytest.mark.parametrize("i", range(len(THIN_CASES) + len(STEM_CASES)))
def test_thin_and_stem_epilogue(eng, i):
    s = (THIN_CASES + STEM_CASES)[i]
    run_case(eng, spec(**s), 4000 + i)


# ---------------------------------------------------------------------------------------------------------------------------------
# out_sv: the epilogue also stores the result as bf16 hi / mid at a channel offset of a halo'd split tensor
def out_sv_buffers(c, pitch, coff, halo):
    n, Ho, Wo = c.s["n"], c.Ho, c.Wo
    shape = (n, Ho + 2 * halo, Wo + 2 * halo, pitch)
    hi = torch.full(shape, SENT16, dtype=torch.int16, device="cuda")
    mid = torch.full(shape, SENT16, dtype=torch.int16, device="cuda")
    sv = c.d.out_sv
    sv.hi, sv.mid, sv.C, sv.Hp, sv.Wp, sv.pt, sv.pl, sv.coff = hi.data_ptr(), mid.data_ptr(), pitch, shape[1], shape[2], halo, halo, coff
    inside = torch.zeros(shape, dtype=torch.bool)
    inside[:, halo:halo + Ho, halo:halo + Wo, coff:coff + c.s["cout"]] = True
    return hi, mid, inside


OUT_SV_CASES = [
    # (spec, os prologue: None / "pow2" / "general", relu, fp32 out written, expected vec2)
    (dict(ALL, act=RELU), None, 0, True, 1),
    (dict(ALL, act=GELU), "pow2", 1, True, 1),
    (dict(scale=True, scale4=True, add1=True, act=SIGMOID), "pow2", 1, True, 0),       # scalar branch's split
    (dict(ALL, act=SILU), "general", 0, True, 1),
    (dict(ALL, act=NONE), "pow2", 1, False, 1),                                        # out.p == NULL: operands only
    (dict(mul1=True, act=SIGMOID2, k=1), None, 0, False, 1),
]


@pytest.mark.parametrize("i", range(len(OUT_SV_CASES)))
def test_out_sv(eng, i):
    kw, os_mode, os_relu, with_out, vec2 = OUT_SV_CASES[i]
    s = spec(**kw, vec2=vec2)
    c = Conv(s, 5000 + i)
    hi, mid, inside = out_sv_buffers(c, 264, 64, 1)
    g = torch.Generator().manual_seed(5100 + i)
    cout = s["cout"]
    os_s = os_t = None
    if os_mode:
        os_s = (2.0 ** torch.randint(-2, 3, (cout,), generator=g)).float() * torch.sign(torch.randn(cout, generator=g))
        if os_mode == "general":
            os_s = os_s * (torch.rand(cout, generator=g) + 0.5)
        os_t = torch.randn(cout, generator=g)
        c.d.os_scale, c.d.os_shift, c.d.os_relu = c.dev(os_s), c.dev(os_t), os_relu
    if not with_out:
        c.d.out = None
    info = launch(eng, c.d)
    if not with_out:
        assert torch.all(c.out.cpu().view(torch.int32) == SENT32), "out_sv: fp32 output written although out.p is NULL"
    expect_path(s, info)
    ref, bound = c.reference(info)
    hic, midc = hi.cpu(), mid.cpu()
    assert torch.all(hic[~inside] == SENT16) and torch.all(midc[~inside] == SENT16), "out_sv: write outside the interior slice"
    sl = (slice(None), slice(1, 1 + c.Ho), slice(1, 1 + c.Wo), slice(64, 64 + cout))
    got_hi, got_mid = hic[sl].permute(0, 3, 1, 2), midc[sl].permute(0, 3, 1, 2)
    if with_out:
        c.check_out(ref, bound, "out_sv")
        y32 = c.y().to(torch.float32)
        if os_mode in (None, "pow2"):
            # the device's fmaf(v, s, t) rounds once; v * 2^k is exact, so the float32 host sum rounds the same way
            v = y32 if os_mode is None else y32 * os_s[None, :, None, None] + os_t[None, :, None, None]
            if os_relu:
                v = v.clamp_min(0)
            want_hi, want_mid = host_split(v)
            assert torch.equal(got_hi, want_hi) and torch.equal(got_mid, want_mid), "out_sv: hi / mid differ from the split of out"
            return
    # general scale or no fp32 output: hi + mid against the float64 chain within the bound, carried through the os prologue
    if os_mode:
        s64, t64 = os_s.to(torch.float64)[None, :, None, None], os_t.to(torch.float64)[None, :, None, None]
        ref_os = ref * s64 + t64
        bound = bound * s64.abs() + ulp32(ref_os)
        if os_relu:
            ref_os = ref_os.clamp_min(0)
        ref = ref_os
    got = split_value(got_hi, got_mid)
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    assert torch.all(err <= bound + 2.0 ** -16 * ref.abs() + 1e-30), f"out_sv: error {err.max().item():.3g}"


# ---------------------------------------------------------------------------------------------------------------------------------
def in_sv_buffers(c, x_nchw, pitch, coff, halo):
    """host-built split of x (float32 NCHW), reflect-haloed, at channels [coff, coff + C) of a wider tensor"""
    n, C, H, W = x_nchw.shape
    xp = F.pad(x_nchw, (halo,) * 4, mode="reflect") if halo else x_nchw
    hi, mid = host_split(xp.permute(0, 2, 3, 1))
    Hi = torch.full((n, H + 2 * halo, W + 2 * halo, pitch), SENT16, dtype=torch.int16)
    Mi = Hi.clone()
    Hi[..., coff:coff + C], Mi[..., coff:coff + C] = hi, mid
    Hi, Mi = Hi.cuda(), Mi.cuda()
    c.keep += [Hi, Mi]
    return Hi, Mi


@pytest.mark.parametrize("mode", [0, 1])
def test_in_sv_matches_internal_split(eng, mode):
    """A pre-split input (host split, reflect halo, channel offset 64 of 192) gives bit for bit what the TMA path computes from the
    fp32 input with its own split pass - which pins in_sv's halo / offset indexing and launch_split's reflect halo together."""
    s = spec(**ALL, act=GELU, mode=mode, h=14, w=22, cout=128)
    c = Conv(s, 6000 + mode)
    info = launch(eng, c.d)
    expect_path(s, info)
    ref, bound = c.reference(info)
    c.check_out(ref, bound, "fp32 input")
    dense = c.out.cpu()
    halo = 1 if mode == 1 else 0
    hi, mid = in_sv_buffers(c, c.x64.to(torch.float32), 192, 64, halo)
    c.out.view(torch.int32).fill_(SENT32)
    sv = c.d.in_sv
    sv.hi, sv.mid, sv.C, sv.Hp, sv.Wp, sv.pt, sv.pl, sv.coff = hi.data_ptr(), mid.data_ptr(), 192, hi.shape[1], hi.shape[2], halo, halo, 64
    c.d.x = None
    info2 = launch(eng, c.d)
    assert KERNELS[info2.kernel] == "tma" and info2.bn == info.bn
    assert torch.equal(c.out.cpu().view(torch.int32), dense.view(torch.int32)), "in_sv result differs from the internal split's"


def test_seg2_ffc_like(eng):
    """FFC's fused GEMM: a 1x1 segment over a pre-split U (channels 64..191 of 192) and a 3x3 reflect segment over a reflect-haloed
    pre-split X (channels 128..255 of 256) accumulate into one tile, then BN scale / shift, ReLU and the block residual."""
    s = spec(cin=128, k=1, cout=256, h=16, w=24, scale=True, add1=dict(cs=384, coff=128), act=RELU, vec2=1)
    c = Conv(s, 6100)
    g = torch.Generator().manual_seed(6101)
    u = c.x64.to(torch.float32)
    x2 = torch.randn(1, 128, 16, 24, generator=g)
    w2 = torch.randn(256, 128, 3, 3, generator=g) / (128 * 9) ** 0.5
    uh, um = in_sv_buffers(c, u, 192, 64, 0)
    xh, xm = in_sv_buffers(c, x2, 256, 128, 1)
    d = c.d
    d.x = None
    d.in_sv.hi, d.in_sv.mid, d.in_sv.C, d.in_sv.Hp, d.in_sv.Wp, d.in_sv.coff = uh.data_ptr(), um.data_ptr(), 192, 16, 24, 64
    d.seg2.hi, d.seg2.mid, d.seg2.C, d.seg2.Hp, d.seg2.Wp, d.seg2.pt, d.seg2.pl, d.seg2.coff = xh.data_ptr(), xm.data_ptr(), 256, 18, 26, 1, 1, 128
    d.seg2_wt = c.dev(w2)
    d.seg2_cin, d.seg2_kh, d.seg2_kw, d.seg2_pad, d.seg2_pad_mode = 128, 3, 3, 1, 1
    info = launch(eng, d)
    expect_path(s, info)
    # the operands are exactly hi + mid of the inputs
    ue = split_value(uh.cpu()[..., 64:192], um.cpu()[..., 64:192]).permute(0, 3, 1, 2)
    xe = split_value(xh.cpu()[:, 1:17, 1:25, 128:256], xm.cpu()[:, 1:17, 1:25, 128:256]).permute(0, 3, 1, 2)
    w1, w2d = c.wt.to(torch.float64), w2.to(torch.float64)
    acc = F.conv2d(ue, w1) + conv64(xe, w2d, 1, 1, 1, 1)
    A = F.conv2d(ue.abs(), w1.abs()) + conv64(xe.abs(), w2d.abs(), 1, 1, 1, 1)
    ref, bound = c.reference(info, acc, A, 128 + 128 * 9)
    c.check_out(ref, bound, "seg2")


def test_strided_grid_tma(eng):
    """oy_mul = ox_mul = 2 phase write (a transposed conv's sub-pixel phase) on the TMA path: the off-phase pixels stay untouched."""
    run_case(eng, spec(**ALL, grid2=True, act=RELU, vec2=1), 6200)
    run_case(eng, spec(**ALL, grid2=True, act=SIGMOID, out_planar=True, vec2=0), 6201)


def test_need_px_skips_only_unneeded_tiles(eng):
    """Output-tile skipping: every element is the sentinel or bit-identical to the dense run, every needed pixel is identical."""
    s = spec(**ALL, act=GELU, h=40, w=48, cout=96)
    c = Conv(s, 6300)
    info = launch(eng, c.d)
    ref, bound = c.reference(info)
    c.check_out(ref, bound, "dense")
    dense = c.out.cpu().view(torch.int32).clone()
    need = torch.zeros(1, c.Ho, c.Wo, dtype=torch.uint8)
    need[0, 3, 5] = 1
    need[0, 30:33, 40:44] = 1
    c.out.view(torch.int32).fill_(SENT32)
    nd = need.cuda()
    c.d.need_px = nd.data_ptr()
    info2 = launch(eng, c.d)
    assert KERNELS[info2.kernel] == "tma"
    sparse = c.out.cpu().view(torch.int32)
    assert torch.all((sparse == dense) | (sparse == SENT32)), "need_px: a written element differs from the dense run"
    y = sel(sparse, False, 0, 96, c.phase, c.Ho, c.Wo)
    yd = sel(dense, False, 0, 96, c.phase, c.Ho, c.Wo)
    m = need[:, None].expand_as(y).bool()
    assert torch.equal(y[m], yd[m]), "need_px: a needed pixel was not written"
    assert (sparse == SENT32).sum() > 0, "need_px: nothing was skipped"


def test_split_reuse_cache(eng):
    """Two sibling TMA convs over one input in one call reuse the operand split; a new call after the host rewrote the input
    does not (the API boundary invalidates the cache), and computes from the new values."""
    s = spec(**ALL, act=RELU, cout=128)
    c = Conv(s, 6400)
    c.d.runs = 2
    info = launch(eng, c.d)
    assert info.convs == 2 and info.split_reused == 1, (info.convs, info.split_reused)
    ref, bound = c.reference(info)
    c.check_out(ref, bound, "siblings")
    c.d.runs = 1
    c.xb.copy_(torch.randn(c.xb.shape, generator=torch.Generator().manual_seed(6401)))
    c.x64 = c.xb.cpu()[..., :64].permute(0, 3, 1, 2).to(torch.float64)
    c.out.view(torch.int32).fill_(SENT32)
    info2 = launch(eng, c.d)
    assert info2.convs == 1 and info2.split_reused == 0
    ref2, bound2 = c.reference(info2)
    c.check_out(ref2, bound2, "rewritten input")


def test_hook_rejects_bad_descriptors(eng):
    from mit_b200 import MitbError
    c = Conv(spec(cout=128), 6500)
    c.d.force_bn = 96                          # 96 is not an N tile choose_bn would consider for Cout 128
    with pytest.raises(MitbError, match="candidate"):
        launch(eng, c.d)
    c.d.force_bn = 0
    c.d.add0.p, c.d.add0.cs = c.d.out + 4, 128
    with pytest.raises(MitbError, match="aligned"):
        launch(eng, c.d)
    c.d.add0.p = None
    c.d.path = PATHS["simt"]
    c.d.out_sv.hi = c.d.out_sv.mid = c.d.out
    with pytest.raises(MitbError, match="TMA path"):
        launch(eng, c.d)


def test_zz_coverage():
    """The cases above reached every kernel, every conv_tma_kernel instantiation and both epilogue branches."""
    if len(RAN) < len(TMA_CASES) + len(GATHER_CASES) + len(SIMT_CASES) + len(THIN_CASES) + len(STEM_CASES) + 2:
        pytest.skip("only part of the module ran")
    kernels = {t[0] for t in TRACES}
    assert kernels >= {"simt", "fewout", "thin", "gather", "gather_splitk", "tma", "stem8"}, kernels
    assert {t[1] for t in TRACES if t[0] == "simt"} == {64, 128}
    inst = {(t[3], t[1]) for t in TRACES if t[0] == "tma"}
    want = {(a, bn) for a in (NONE, RELU, GELU, SILU, -1) for bn in (32, 64, 96, 128)}
    assert inst >= want, sorted(want - inst)
    for a in (NONE, RELU, GELU, SILU, -1):
        for bn in (32, 64, 96, 128):
            assert {t[2] for t in TRACES if t[0] == "tma" and t[3] == a and t[1] == bn} == {0, 1}, (a, bn)
    assert {t[2] for t in TRACES if t[0] == "gather"} == {0, 1}
    assert any(t[0] == "gather_splitk" and t[4] > 1 for t in TRACES)
    print("conv epilogue coverage:", sorted({t[:4] for t in TRACES}))

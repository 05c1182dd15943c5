"""The two kernels the OCR's characters come out of, against torch float64 on the CPU (never another kernel of the library).

Vocabulary head (test hook mitb_test_vocab_head): logits = x wt^T + bias with log-softmax and argmax fused into the GEMM's
epilogue, per row the first maximal column (torch's log_softmax(2).max(2), model_48px_ctc.py:459-460) and its log-probability.
Every kernel writes per-row (max, first argmax, sum exp(v - max)) partials per column block, and rowstat_final merges them.

* Exact cases: x small integers (|x| <= 3), weights and bias multiples of 1/8 with |w| <= 2.  Every product and partial sum is
  exact in fp32 and in the bf16 hi / mid split (the mid is 0), so every kernel's logits are the float64 logits and idx must be
  the first maximal column on every row, with no "safe margin" filter.  Tie rows are one-hot x rows against duplicated weight
  rows, placed so that the two maxima meet at each merge level (see tie_pairs).  The partials are checked block by block.
* Real-valued cases: the logit error bound of test_gpu_conv_epilogue.py, E_c = c * A_c + ulp(v_c) with A = |x| |wt|^T in float64
  (tensor cores, bf16x3 split: c = 2^-15; SIMT fp32: c = (C + 2) * 2^-24) and one ulp for the bias add.  The log-probability
  v_max - logsumexp(v) moves by at most 2 max_c E_c through the logits.  The fp32 exp / sum / log chain adds
  rho = 2^-24 (4 L + 3 (ln V + 3)) relatively to the sum (L: the longest chain of sequential add / rescale / exp steps a
  column's term goes through: the columns of one thread, the lane merges, the blocks of one rowstat_final lane and its 5
  shuffle levels, each at most 4 ulp; ln V + 3 bounds the weighted mean rounding of the exp arguments, once per level), and
  2 ulp of the result for the log.  idx must be a column whose float64 logit is within E_idx + E_max of the maximum, which is
  the reference's argmax wherever the float64 top-2 gap exceeds the bounds.

Attention core (mitb_op_attention): softmax(q k^T / sqrt(hd)) v per (line, head).  A score's fp32 error is at most
delta = gamma_{hd+1} scale sum_d |q_d| |k_d| (hd fused multiply-adds and the scale), which moves each probability by at most
2 delta_max relatively; the fp32 exp, sum, rescale and P.V accumulation add rho = 2^-24 (2 T + 2 (ln T + 5) + 8) relatively.  So
|out_d - ref_d| <= (2 delta_max + rho) sum_j p_j |v_jd| + 2 ulp(ref_d).  T covers attention40_kernel (hd 40, 16-byte aligned,
T <= 416), the generic kernel (T >= 417, hd != 40, unaligned operands) and its key blocks of 64 (T = 64, 65, 129).

The last test asserts that the head cases reached all three kernels and every N tile."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

KERNELS = {1: "simt", 4: "gather", 6: "tma"}
PATHS = {"simt": 1, "gather": 2, "tma": 3}
SENT32 = 0x7FC0DEAD            # fp32 NaN with a payload no kernel produces
SENTI = -0x21524111            # int32 sentinel
TAIL = 37                      # sentinel elements past every buffer's written range
INT_MAX = 2 ** 31 - 1
TRACES = []                    # (kernel, bn) of every head call of this module


@pytest.fixture(scope="module")
def eng():
    from mit_b200.engine import get_engine
    return get_engine("cuda:0")


def ulp32(v):
    _, e = torch.frexp(v.abs().to(torch.float64))
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 24)


def pick_bn(V):
    """the tensor-core N tile of a V-column weight (conv_tc.cu pick_bn)"""
    tiles = (V + 127) // 128
    return max(32, (-(-V // tiles) + 31) // 32 * 32)


def layout(V, path):
    """(blocks per row, columns per block) of the row-stat partials: two halves per N tile on the tensor cores, 128 on SIMT"""
    if path == "simt":
        return (V + 127) // 128, 128
    bn = pick_bn(V)
    return 2 * (-(-V // bn)), bn // 2


def first_argmax(v):
    """first maximal column of each row (float64, exact comparison)"""
    cols = torch.arange(v.shape[1]).expand_as(v)
    return torch.where(v == v.max(1, keepdim=True).values, cols, v.shape[1]).min(1).values


def run_head(eng, x, wt, bias, path):
    """mitb_test_vocab_head with sentinel-filled outputs and partial buffers; returns (idx, logprob, pmax, psum, pidx, info, nblk)"""
    from mit_b200 import _lib as L
    rows, V = x.shape[0], wt.shape[0]
    nb, _ = layout(V, path)
    cap = rows * nb
    idx = torch.full((rows + TAIL,), SENTI, dtype=torch.int32, device="cuda")
    lp = torch.full((rows + TAIL,), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    pmax = torch.full((cap + TAIL,), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    psum = pmax.clone()
    pidx = torch.full((cap + TAIL,), SENTI, dtype=torch.int32, device="cuda")
    xd, wd = x.to(torch.float32).contiguous().cuda(), wt.to(torch.float32).contiguous().cuda()
    bd = bias.to(torch.float32).contiguous().cuda() if bias is not None else None
    info, nblk = L.MitbTestConvInfo(), C.c_int32()
    n, t = (3, rows // 3) if rows % 3 == 0 else (1, rows)
    eng._call(eng.lib.mitb_test_vocab_head, xd.data_ptr(), n, t, x.shape[1], wd.data_ptr(), bd.data_ptr() if bd is not None else None,
              V, PATHS[path], idx.data_ptr(), lp.data_ptr(), pmax.data_ptr(), psum.data_ptr(), pidx.data_ptr(), cap + TAIL,
              C.byref(nblk), C.byref(info), eng._stream())
    torch.cuda.synchronize()
    TRACES.append((KERNELS.get(info.kernel, "?"), info.bn))
    assert KERNELS.get(info.kernel) == path, (path, info.kernel)
    assert nblk.value == nb, (nblk.value, nb)
    if path != "simt":
        assert info.bn == pick_bn(V), (info.bn, pick_bn(V))
    idx, lp, pmax, psum, pidx = (b.cpu() for b in (idx, lp, pmax, psum, pidx))
    assert torch.all(idx[rows:] == SENTI) and torch.all(lp[rows:].view(torch.int32) == SENT32), "write past n*T rows"
    assert torch.all(pidx[cap:] == SENTI) and torch.all(pmax[cap:].view(torch.int32) == SENT32) and \
        torch.all(psum[cap:].view(torch.int32) == SENT32), "partials written past n*T rows"
    return (idx[:rows].long(), lp[:rows].to(torch.float64), pmax[:cap].view(rows, nb), psum[:cap].view(rows, nb),
            pidx[:cap].view(rows, nb), info, nb)


def chain_rho(V, path, nb):
    """relative bound of the fp32 exp / sum chain (module docstring)"""
    per_thread = 8 if path == "simt" else pick_bn(V) // 4
    lanes = 4 if path == "simt" else 2
    L = per_thread + lanes + -(-nb // 32) + 5
    return 2.0 ** -24 * (4 * L + 3 * (math.log(V) + 3))


def block_stats(v, nb, width):
    """float64 (max, first argmax, sum exp(v - max)) of each column block; empty blocks (-inf, INT_MAX, 0)"""
    rows, V = v.shape
    pad = torch.full((rows, nb * width), -math.inf, dtype=torch.float64)
    pad[:, :V] = v
    b = pad.view(rows, nb, width)
    m = b.max(2).values
    cols = torch.arange(nb * width).view(nb, width).expand(rows, nb, width)
    i = torch.where((b == m[..., None]) & (b > -math.inf), cols, INT_MAX).min(2).values
    s = torch.where(m[..., None] > -math.inf, torch.exp(b - m[..., None]), torch.zeros_like(b)).sum(2)
    return m, i, s


def tie_pairs(V):
    """column pairs (a < b) whose logits tie at each merge level the kernels have, for a V-column head"""
    bn = pick_bn(V)
    half = bn // 2
    want = [
        (0, 8),                         # one thread of the tensor-core epilogue (8 columns apart)
        (1, 7),                         # across its 4 lanes, lower column in the lower lane
        (6, 9),                         # across its 4 lanes, lower column in the higher lane
        (half - 2, half + 1),           # across the two column halves of an N tile
        (3, bn + 3),                    # across N tiles
        (10, 16 * bn + 10),             # rowstat_final blocks 0 and 32 (one lane)
        (half + 6, 16 * bn + 20),       # rowstat_final blocks 1 and 32 (two lanes)
        (4, 68),                        # SIMT: one thread's j < 4 and j >= 4 columns
        (2, 5),                         # SIMT: two threads
        (11, 139),                      # SIMT: two 128-column blocks
        (12, 4096 + 12),                # SIMT: rowstat_final blocks 0 and 32
        (141, 4096 + 30),               # SIMT: rowstat_final blocks 1 and 32
        (13, V - 1),                    # the last column
    ]
    used, pairs = set(), []
    for a, b in want:
        if b < V and a not in used and b not in used and a != b:
            pairs.append((a, b))
            used |= {a, b}
    return pairs


def exact_case(V, C, rows, seed, const_bias=False):
    """(x, wt, bias, tie rows) with exact fp32 / bf16x3 logits; tie rows are one-hot x rows whose maximum is a duplicated pair"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, (rows, C), generator=g).to(torch.float64)
    wt = torch.randint(-16, 16, (V, C), generator=g).to(torch.float64) / 8          # |w| <= 1.875 except the tie channels
    bias = torch.randint(-16, 16, (V,), generator=g).to(torch.float64) / 8
    ties = []
    if const_bias:
        bias[:] = 1.25
        x[::5] = 0                      # all-equal rows
        return x, wt, bias, ties
    for k, (a, b) in enumerate(tie_pairs(V)):
        assert k < C
        wt[b] = wt[a]
        wt[a, k] = wt[b, k] = 2.0
        bias[a] = bias[b] = 2.0         # 3 * 2 + 2 = 8 > 3 * 1.875 + 2: the pair is the row's only maximum
        r = (7 * k + 1) % rows
        x[r] = 0
        x[r, k] = 3
        ties.append((r, a))
    return x, wt, bias, ties


def logits64(x, wt, bias):
    v = x @ wt.T
    return v + bias if bias is not None else v


HEAD_V = [20, 40, 150, 448, 512, 46000]
HEAD_PATHS = ["simt", "gather", "tma"]


@pytest.mark.parametrize("path", HEAD_PATHS)
@pytest.mark.parametrize("V", HEAD_V)
def test_vocab_head_exact(eng, V, path):
    """exact logits: idx is the first maximal column on every row (ties included), logprob and partials within the chain bound"""
    rows, C = 171, 320                  # 3 lines x 57 steps: a ragged last M tile
    x, wt, bias, ties = exact_case(V, C, rows, 1000 + V)
    idx, lp, pmax, psum, pidx, info, nb = run_head(eng, x, wt, bias, path)
    v = logits64(x, wt, bias)
    ref_idx = first_argmax(v)
    for r, a in ties:
        assert ref_idx[r] == a
    bad = (idx != ref_idx).nonzero().flatten()
    assert bad.numel() == 0, f"V={V} {path}: idx differs on {bad.numel()} rows, e.g. row {bad[0].item()}: {idx[bad[0]].item()} vs {ref_idx[bad[0]].item()}"
    ref_lp = torch.log_softmax(v, 1).max(1).values
    rho = chain_rho(V, path, nb)
    err = (lp - ref_lp).abs()
    bound = rho + 2 * ulp32(ref_lp)
    assert torch.all(err <= bound), f"V={V} {path}: logprob err {err.max().item():.3e}, ratio {(err / bound).max().item():.2f}"
    # partials, block by block: max and first argmax exact, sum within the chain bound
    _, width = layout(V, path)
    m, i, s = block_stats(v, nb, width)
    assert torch.equal(pmax.to(torch.float64), m), f"V={V} {path}: block max"
    assert torch.equal(pidx.long(), i), f"V={V} {path}: block argmax"
    serr = (psum.to(torch.float64) - s).abs()
    assert torch.all(serr <= rho * s), f"V={V} {path}: block sum err ratio {(serr / (rho * s).clamp_min(1e-300)).max().item():.2f}"
    print(f"exact V={V} {path}: bn {info.bn} nblk {nb} ties {len(ties)} lp bound ratio {(err / bound).max().item():.3f}")


@pytest.mark.parametrize("path", HEAD_PATHS)
@pytest.mark.parametrize("V", [40, 448, 46000])
def test_vocab_head_all_equal(eng, V, path):
    """x = 0 with a constant bias: every logit equal, idx 0 and logprob within one ulp of -log V"""
    x, wt, bias, _ = exact_case(V, 320, 171, 2000 + V, const_bias=True)
    idx, lp, _, _, _, _, _ = run_head(eng, x, wt, bias, path)
    v = logits64(x, wt, bias)
    assert torch.equal(idx, first_argmax(v))
    eq = (x == 0).all(1)
    assert torch.all(idx[eq] == 0)
    want = torch.full_like(lp[eq], -math.log(V))
    assert torch.all((lp[eq] - want).abs() <= ulp32(want)), (lp[eq] - want).abs().max().item()


def real_case(V, C, rows, seed, spread, dominant):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, C, generator=g)
    wt = torch.randn(V, C, generator=g) * (spread / C ** 0.5)
    bias = torch.randn(V, generator=g)
    if dominant:                        # every 4th row: one column far above the rest (logprob ~ 0)
        for r in range(0, rows, 4):
            c = (r * 7919) % V
            x[r] = 3 * torch.sign(wt[c])
    return x, wt, bias


@pytest.mark.parametrize("path", HEAD_PATHS)
@pytest.mark.parametrize("V,C,spread,dominant,nobias", [
    (20, 320, 1.0, False, False), (40, 320, 1.0, True, False), (150, 256, 1.0, False, True), (448, 320, 60.0, False, False),
    (512, 256, 1.0, True, False), (46000, 320, 1.0, True, False), (46000, 256, 60.0, False, False)])
def test_vocab_head_real(eng, V, C, spread, dominant, nobias, path):
    """real-valued logits (spread 60: about +-200): logprob within the derived bound, idx within the candidates of the bound"""
    rows = 171 if V < 46000 else 300
    x, wt, bias = real_case(V, C, rows, 3000 + V + C, spread, dominant)
    if nobias:
        bias = None
    idx, lp, pmax, _, _, info, nb = run_head(eng, x, wt, bias, path)
    x64, w64 = x.to(torch.float64), wt.to(torch.float64)
    v = logits64(x64, w64, bias.to(torch.float64) if bias is not None else None)
    A = x64.abs() @ w64.abs().T
    c = 2.0 ** -15 if path != "simt" else (C + 2) * 2.0 ** -24
    E = c * A + (ulp32(v) if bias is not None else 0)
    vmax = v.max(1).values
    ref_idx = first_argmax(v)
    ok = v.gather(1, idx[:, None])[:, 0] >= vmax - E.gather(1, idx[:, None])[:, 0] - E.gather(1, ref_idx[:, None])[:, 0]
    assert ok.all(), f"V={V} {path}: idx outside the candidates on {(~ok).sum().item()} rows"
    top2 = v.topk(2, 1).values
    sure = (top2[:, 0] - top2[:, 1]) > 2 * E.max(1).values
    assert torch.equal(idx[sure], ref_idx[sure])
    ref_lp = torch.log_softmax(v, 1).max(1).values
    bound = 2 * E.max(1).values + chain_rho(V, path, nb) + 2 * ulp32(ref_lp)
    err = (lp - ref_lp).abs()
    assert torch.all(err <= bound), f"V={V} {path}: logprob err {err.max().item():.3e}, ratio {(err / bound).max().item():.2f}"
    _, width = layout(V, path)
    m, _, _ = block_stats(v, nb, width)
    Eb = torch.full((rows, nb * width), 0.0, dtype=torch.float64)
    Eb[:, :V] = E
    Eb = Eb.view(rows, nb, width).max(2).values
    fin = m > -math.inf
    assert torch.all((pmax.to(torch.float64)[fin] - m[fin]).abs() <= Eb[fin]), f"V={V} {path}: block max"
    assert torch.all(pmax[~fin] == -math.inf)
    print(f"real V={V} C={C} {path}: bn {info.bn} sure rows {int(sure.sum())}/{rows} lp bound ratio {(err / bound).max().item():.3f}")


def test_vocab_head_rejects_small_partials(eng):
    from mit_b200 import MitbError
    from mit_b200 import _lib as L
    x = torch.zeros(171, 320, device="cuda")
    wt = torch.zeros(512, 320, device="cuda")
    out = torch.zeros(1024, device="cuda")
    info, nblk = L.MitbTestConvInfo(), C.c_int32()
    with pytest.raises(MitbError, match="partials"):
        eng._call(eng.lib.mitb_test_vocab_head, x.data_ptr(), 3, 57, 320, wt.data_ptr(), None, 512, PATHS["tma"], out.data_ptr(),
                  out.data_ptr(), out.data_ptr(), out.data_ptr(), out.data_ptr(), 171 * 8 - 1, C.byref(nblk), C.byref(info), eng._stream())


# ---------------------------------------------------------------------------------------------------------------------------------
# attention

def attention_ref(qk, v, n, T, heads, hd):
    """float64 output and its bound (module docstring)"""
    d = heads * hd
    q = qk[:, :d].to(torch.float64).view(n, T, heads, hd).transpose(1, 2)
    k = qk[:, d:].to(torch.float64).view(n, T, heads, hd).transpose(1, 2)
    vv = v.to(torch.float64).view(n, T, heads, hd).transpose(1, 2)
    scale = 1.0 / math.sqrt(hd)
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, -1)
    ref = p @ vv
    u = 2.0 ** -24
    gamma = (hd + 1) * u / (1 - (hd + 1) * u)
    delta = (gamma * scale * (q.abs() @ k.abs().transpose(-1, -2))).amax(-1, keepdim=True)
    rho = u * (2 * T + 2 * (math.log(T) + 5) + 8)
    mag = p @ vv.abs()
    bound = (2 * delta + rho) * mag + 2 * ulp32(ref)
    return (ref.transpose(1, 2).reshape(n * T, d), bound.transpose(1, 2).reshape(n * T, d))


def attention_inputs(n, T, heads, hd, mode, seed):
    g = torch.Generator().manual_seed(seed)
    d = heads * hd
    v = torch.randn(n * T, d, generator=g)
    if mode == "random":                # scores span about +-30
        qk = 3.0 * torch.randn(n * T, 2 * d, generator=g)
    elif mode == "equal":               # q = 0: every score 0, the output is the mean of V
        qk = torch.randn(n * T, 2 * d, generator=g)
        qk[:, :d] = 0
    else:                               # one dominant key per (line, head)
        u = torch.randn(n, 1, heads, hd, generator=g)
        q = u + 0.1 * torch.randn(n, T, heads, hd, generator=g)
        k = 0.1 * torch.randn(n, T, heads, hd, generator=g)
        k[:, (T * 5) // 7] = 4 * u[:, 0]
        qk = torch.cat([q.reshape(n * T, d), k.reshape(n * T, d)], 1)
    return qk, v


def run_attention(eng, qk, v, n, T, heads, hd, offset):
    """mitb_op_attention on device copies whose base pointers are `offset` floats past a 256-byte aligned allocation"""
    def dev(t):
        b = torch.zeros(t.numel() + offset, device="cuda")
        b[offset:].copy_(t.reshape(-1))
        return b
    qkd, vd = dev(qk), dev(v)
    out = torch.full((n * T * heads * hd + TAIL,), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    eng._call(eng.lib.mitb_op_attention, qkd.data_ptr() + 4 * offset, vd.data_ptr() + 4 * offset, n, T, heads, hd, out.data_ptr(),
              eng._stream())
    out = out.cpu()
    assert torch.all(out[n * T * heads * hd:].view(torch.int32) == SENT32), "write past the output"
    return out[:n * T * heads * hd].view(n * T, heads * hd)


ATT_T = [1, 5, 31, 32, 33, 57, 160, 416, 417, 565, 566, 1024, 2048]


def att_lines(T):
    return max(1, min(16, (1 << 24) // (8 * T * T)))


def check_attention(eng, T, hd, mode, offset, seed):
    n, heads = att_lines(T), 8
    qk, v = attention_inputs(n, T, heads, hd, mode, seed)
    out = run_attention(eng, qk, v, n, T, heads, hd, offset)
    ref, bound = attention_ref(qk, v, n, T, heads, hd)
    assert torch.isfinite(out).all()
    err = (out.to(torch.float64) - ref).abs()
    ratio = (err / bound).max().item()
    assert torch.all(err <= bound), f"attention n={n} T={T} hd={hd} {mode} offset={offset}: max err {err.max().item():.3e}, ratio {ratio:.2f}"
    print(f"attention n={n} T={T} hd={hd} {mode} offset={offset}: bound ratio {ratio:.3f}")


@pytest.mark.parametrize("mode", ["random", "equal", "dominant"])
@pytest.mark.parametrize("T", ATT_T)
def test_attention_hd40(eng, T, mode):
    """the OCR encoder's shape (8 heads of 40), aligned operands: attention40_kernel up to T = 416, the streamed kernel above"""
    check_attention(eng, T, 40, mode, 0, 100 + T)


@pytest.mark.parametrize("T", [1, 33, 64, 65, 129, 417, 2048])
@pytest.mark.parametrize("hd,offset", [(40, 1), (32, 0), (64, 0)])
def test_attention_generic(eng, T, hd, offset):
    """the generic kernel: hd 40 at a 4-byte offset (not 16-byte aligned), hd 32 and 64; key blocks of 64 (T 64, 65, 129)"""
    check_attention(eng, T, hd, "random", offset, 200 + T + hd)
    if T in (65, 2048):
        check_attention(eng, T, hd, "dominant", offset, 300 + T + hd)


def test_zz_coverage():
    """The head cases reached all three kernels and every N tile on both tensor-core kernels."""
    if len(TRACES) < len(HEAD_V) * len(HEAD_PATHS) * 2:
        pytest.skip("only part of the module ran")
    assert {t[0] for t in TRACES} == {"simt", "gather", "tma"}
    for k in ("gather", "tma"):
        assert {t[1] for t in TRACES if t[0] == k} == {32, 64, 96, 128}, k
    assert {t[1] for t in TRACES if t[0] == "simt"} == {128}

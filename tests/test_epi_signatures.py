"""Which kernel each staged TMA conv launch of a bench page runs (conv_tma.cu: MITB_EPI_SIGS, staged_epi_sig), without a GPU.

tests/golden/conv_epi_launches_1page.txt lists the TMA conv launches of one 2048x1536 page with their activation instantiation and
the parts of their fused chain.  Every staged launch of that page must map to the kernel of its own signature (the runtime-switch
activation, two tiny launches, excepted), every instantiated signature must occur on the page, and anything else - other part
combinations, or all of them with specialisation switched off - must map to the generic signature."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GENERIC = 512
ADD0, SCALE, SHIFT, MUL1, ADD1, OUT, OS, OS_AFFINE, OS_RELU = 1, 2, 4, 8, 16, 32, 64, 128, 256
NONE, RELU, GELU, SILU = 0, 1, 2, 3


@pytest.fixture(scope="module")
def lib():
    from mit_b200 import _lib
    return _lib.load()


def page_launches():
    rows = []
    for ln in open(os.path.join(ROOT, "tests", "golden", "conv_epi_launches_1page.txt")):
        if ln.startswith("#") or not ln.strip():
            continue
        m, k, n, bn, nkb, act, parts, staged = (int(x) for x in ln.split())
        rows.append(dict(M=m, K=k, N=n, BN=bn, nkb=nkb, act=act, parts=parts, staged=staged))
    return rows


def instantiated(lib):
    n = lib.mitb_test_epi_signatures(None, None, 0)
    act, sig = (C.c_int * n)(), (C.c_int * n)()
    assert lib.mitb_test_epi_signatures(act, sig, n) == n
    return set(zip(act, sig))


def test_page_launches_run_their_own_signature(lib):
    rows = page_launches()
    staged = [r for r in rows if r["staged"]]
    assert len(rows) > 300 and len(staged) > 200
    for r in staged:
        want = GENERIC if r["act"] == -1 else r["parts"]
        assert lib.mitb_test_epi_signature(r["act"], r["parts"]) == want, r
    used = {(r["act"], r["parts"]) for r in staged}
    assert instantiated(lib) <= used, "an instantiated signature no staged launch of the page has"


def test_other_combinations_fall_back_to_generic(lib):
    sigs = instantiated(lib)
    for act in (NONE, RELU, GELU, SILU, -1):
        for parts in range(1, GENERIC):
            if parts & (OS_AFFINE | OS_RELU) and not parts & OS or parts & OS_RELU and not parts & OS_AFFINE:
                continue                                   # the split's prologue exists only with a split output
            want = parts if (act, parts) in sigs else GENERIC
            assert lib.mitb_test_epi_signature(act, parts) == want, (act, parts)
    for parts in (ADD0 | SHIFT | OUT, SCALE | SHIFT | MUL1 | ADD1 | OUT | OS, SHIFT | OS | OS_AFFINE):
        assert lib.mitb_test_epi_signature(GELU, parts) == GENERIC


def test_switch_forces_generic(lib):
    prev = lib.mitb_set_epi_specialise(0)
    try:
        for act, parts in instantiated(lib):
            assert lib.mitb_test_epi_signature(act, parts) == GENERIC
    finally:
        lib.mitb_set_epi_specialise(prev)
    assert lib.mitb_set_epi_specialise(prev) == prev
    on = lib.mitb_test_epi_signature(GELU, SHIFT | OS)
    assert on == (SHIFT | OS if prev else GENERIC)

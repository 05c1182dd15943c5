"""ctypes binding of libmitb.so (C ABI declared in include/mitb.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``csrc/Makefile``.  There is no fallback: if the
shared object is missing, or no Hopper (sm_90a) GPU is visible, loading / context creation raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmitb.so")


class MitbTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("ndim", C.c_int32), ("shape", C.c_int64 * 4)]


class MitbTestView(C.Structure):
    _fields_ = [("p", C.c_void_p), ("cs", C.c_int32), ("coff", C.c_int32), ("planar", C.c_int32), ("reserved", C.c_int32)]


class MitbTestSplit(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("mid", C.c_void_p), ("C", C.c_int32), ("Hp", C.c_int32), ("Wp", C.c_int32),
                ("pt", C.c_int32), ("pl", C.c_int32), ("coff", C.c_int32)]


def _ints(*names):
    return [(n, C.c_int32) for n in names]


class MitbTestConvDesc(C.Structure):
    """mitb_test_conv_desc (test hook, include/mitb.h): one fully described conv with every fused-epilogue option."""
    _fields_ = ([("x", C.c_void_p)] + _ints("N", "H", "W", "C", "cs", "coff", "planar", "in_relu") +
                [("in_scale", C.c_void_p), ("in_shift", C.c_void_p), ("wt", C.c_void_p)] +
                _ints("cout", "wt_cin", "kh", "kw", "stride", "pad_y", "pad_x", "pad_mode") +
                [("scale", C.c_void_p), ("shift", C.c_void_p), ("mul1", C.c_void_p)] + _ints("act", "runs") +
                [("add0", MitbTestView), ("add1", MitbTestView), ("out", C.c_void_p)] +
                _ints("out_H", "out_W", "out_cs", "out_coff", "out_planar", "oy_mul", "oy_add", "ox_mul", "ox_add", "reserved0") +
                [("out_sv", MitbTestSplit), ("os_scale", C.c_void_p), ("os_shift", C.c_void_p)] + _ints("os_relu", "reserved1") +
                [("in_sv", MitbTestSplit), ("seg2", MitbTestSplit), ("seg2_wt", C.c_void_p)] +
                _ints("seg2_cin", "seg2_kh", "seg2_kw", "seg2_pad", "seg2_pad_mode", "reserved2") +
                [("need_px", C.c_void_p)] + _ints("path", "force_bn"))


class MitbTestConvInfo(C.Structure):
    _fields_ = _ints("kernel", "bn", "splits", "vec2", "tma_act", "split_reused", "convs", "staged", "epi_sig")


class MitbTestFftDesc(C.Structure):
    """mitb_test_fft_desc (test hook, include/mitb.h): one real 2-D FFT on the planar or the NHWC implementation."""
    _fields_ = (_ints("impl", "inverse", "N", "h", "w", "C") + [("in", MitbTestView), ("out", MitbTestView), ("out_sv", MitbTestSplit),
                                                                ("add", MitbTestView)] + _ints("force_plain", "reserved"))


class MitbTestFftInfo(C.Structure):
    _fields_ = ([("h_nst", C.c_int32), ("h_radix", C.c_int32 * 16), ("w_nst", C.c_int32), ("w_radix", C.c_int32 * 16)] +
                _ints("rows_tma", "rows_box_rows", "cols_tma", "cols_box_rows", "P", "CB"))


class MitbError(RuntimeError):
    pass


_lib = None

# name -> (restype, argtypes); mirrors include/mitb.h one to one (checked by tests/test_host.py::test_abi_header_and_library_agree)
P, I, F, LL, D = C.c_void_p, C.c_int, C.c_float, C.c_longlong, C.c_double
SIGNATURES = {
    "mitb_create": (I, [I, C.POINTER(P)]),
    "mitb_destroy": (None, [P]),
    "mitb_last_error": (C.c_char_p, [P]),
    "mitb_version": (C.c_char_p, []),
    "mitb_launch_count": (C.c_longlong, [P]),
    "mitb_workspace_bytes": (C.c_size_t, [P]),
    "mitb_set_tensor_cores": (I, [I]),
    "mitb_set_ffc_mode": (I, [I]),
    "mitb_set_sparse_decoder": (I, [I]),
    "mitb_profile_enable": (I, [P, I]),
    "mitb_profile_report": (C.c_char_p, [P]),
    "mitb_dbnet_load": (I, [P, C.POINTER(MitbTensor), I]),
    "mitb_dbnet_unload": (I, [P]),
    "mitb_dbnet_forward": (I, [P, P, I, I, I, P, P, P]),
    "mitb_dbnet_forward_u8": (I, [P, P, I, I, I, P, P, P]),
    "mitb_dbnet_r34_load": (I, [P, C.POINTER(MitbTensor), I]),
    "mitb_dbnet_r34_unload": (I, [P]),
    "mitb_dbnet_r34_forward": (I, [P, P, I, I, I, P, P, P]),
    "mitb_dbnet_r34_forward_u8": (I, [P, P, I, I, I, P, P, P]),
    "mitb_ocr_load": (I, [P, C.POINTER(MitbTensor), I]),
    "mitb_ocr_unload": (I, [P]),
    "mitb_ocr_timesteps": (I, [I]),
    "mitb_ocr_forward": (I, [P, P, I, I, P, P, P, P]),
    "mitb_ocr_forward_u8": (I, [P, P, I, I, P, P, P, P]),
    "mitb_lama_load": (I, [P, C.POINTER(MitbTensor), I]),
    "mitb_lama_unload": (I, [P]),
    "mitb_lama_forward": (I, [P, P, P, P, P, I, I, I, P, P]),
    "mitb_lama_forward_mpe256": (I, [P, P, P, P, P, I, I, I, P, P]),
    "mitb_lama_infer_u8": (I, [P, P, P, P, P, I, I, I, P, P]),
    "mitb_op_conv2d": (I, [P, P, I, I, I, I, P, I, I, I, I, I, I, I, I, P, I, P, P, I, P, P]),
    "mitb_op_conv_transpose2d": (I, [P, P, I, I, I, I, P, I, I, I, I, P, I, P, P]),
    "mitb_op_dwconv7_ln": (I, [P, P, I, I, I, I, P, P, P, P, F, P, P]),
    "mitb_op_maxpool3x3s2": (I, [P, P, I, I, I, I, P, P]),
    "mitb_op_layernorm": (I, [P, P, I, I, P, P, F, P, P]),
    "mitb_op_rfft2": (I, [P, P, I, I, I, P, P]),
    "mitb_op_irfft2": (I, [P, P, I, I, I, P, P]),
    "mitb_op_rfft2_nhwc": (I, [P, P, I, I, I, I, P, P]),
    "mitb_op_irfft2_nhwc": (I, [P, P, P, I, I, I, I, P, P]),
    "mitb_op_attention": (I, [P, P, P, I, I, I, I, P, P]),
    "mitb_op_mpe_tables": (I, [P, P, I, P, P, P]),
    "mitb_op_bilateral17": (I, [P, P, I, I, P, P]),
    "mitb_op_warp_lines_u8": (I, [P, P, I, I, P, I, P, I, I, P]),
    "mitb_op_ctc_collapse": (I, [P, P, P, P, I, I, P, P, P, P, P, P]),
    "mitb_op_textline_pairs": (I, [P, P, I, D, D, D, D, D, D, P, P]),
    "mitb_op_resize_linear_u8": (I, [P, P, I, I, I, P, I, I, I, P]),
    "mitb_op_cut_rects": (I, [P, P, I, I, P, I, P]),
    "mitb_op_cc_label": (I, [P, P, I, I, P, P, P, I, P, P]),
    "mitb_op_owner_map": (I, [P, P, P, I, P, P]),
    "mitb_op_crf_workspace": (I, [LL, LL, LL, C.POINTER(C.c_ulonglong)]),
    "mitb_op_dense_crf": (I, [P, P, P, I, P, P, I, I, I, I, LL, LL, LL, I, F, F, F, F, F, F, P, P, P, P]),
    "mitb_op_dilate_lines": (I, [P, P, I, I, P, P, P, I, P, P]),
    "mitb_op_dilate_se": (I, [P, P, I, I, P, I, P, P]),
    "mitb_test_conv": (I, [P, C.POINTER(MitbTestConvDesc), C.POINTER(MitbTestConvInfo), P]),
    "mitb_test_struct_sizes": (I, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mitb_test_vocab_head": (I, [P, P, I, I, I, P, P, I, I, P, P, P, P, P, LL, C.POINTER(C.c_int32), C.POINTER(MitbTestConvInfo), P]),
    "mitb_test_fft": (I, [P, C.POINTER(MitbTestFftDesc), C.POINTER(MitbTestFftInfo), P]),
    "mitb_set_epi_specialise": (I, [I]),
    "mitb_test_epi_signature": (I, [I, I]),
    "mitb_test_epi_signatures": (I, [C.POINTER(C.c_int), C.POINTER(C.c_int), I]),
}


def load():
    """dlopen libmitb.so and attach the prototypes.  Raises if the library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MitbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        f"(nvcc, sm_90a). There is no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib

"""Thin Python host over the C ABI: owns one mitb context per GPU, hands torch CUDA tensors (used purely as device
memory containers) to the library and returns torch tensors.  No arithmetic of the hot path happens in torch."""
from __future__ import annotations

import ctypes as C
import threading
from collections import OrderedDict
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from ._lib import MitbError, MitbTensor


class _Trace:
    """Wall-clock accounting of the host path (MITB_E2E_TRACE=1): seconds per label summed over all threads."""
    import os as _os
    on = bool(int(_os.environ.get("MITB_E2E_TRACE", "0") or 0))
    acc: Dict[str, float] = {}
    cnt: Dict[str, int] = {}
    lock = threading.Lock()

    def __init__(self, label):
        self.label = label

    def __enter__(self):
        if _Trace.on:
            import time
            self.t0 = time.perf_counter()
        return self

    def __exit__(self, *a):
        if _Trace.on:
            import time
            dt = time.perf_counter() - self.t0
            with _Trace.lock:
                _Trace.acc[self.label] = _Trace.acc.get(self.label, 0.0) + dt
                _Trace.cnt[self.label] = _Trace.cnt.get(self.label, 0) + 1


def trace(label):
    return _Trace(label)


def trace_report(reset=True):
    with _Trace.lock:
        r = {k: (round(v, 4), _Trace.cnt[k]) for k, v in sorted(_Trace.acc.items(), key=lambda kv: -kv[1])}
        if reset:
            _Trace.acc.clear()
            _Trace.cnt.clear()
    return r


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class Engine:
    """One context bound to one CUDA device (one process per GPU in multi-GPU runs)."""

    def __init__(self, device="cuda:0"):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise MitbError("mit_b200 needs a CUDA (H100, sm_90a) device; there is no CPU fallback")
        self.device = torch.device(device if str(device) != "cuda" else "cuda:0")
        if self.device.type != "cuda":
            raise MitbError(f"mit_b200 runs on CUDA only, got device '{device}'")
        torch.cuda.set_device(self.device)
        h = C.c_void_p()
        rc = self.lib.mitb_create(self.device.index or 0, C.byref(h))
        if rc != 0:
            raise MitbError(self.lib.mitb_last_error(None).decode())
        self._h = h
        self._keep = {}
        self._lock = threading.RLock()   # the context is not re-entrant: page-pipeline threads serialise their ENQUEUES here
        self._pin_lock = threading.Lock()
        self._pinned = OrderedDict()   # (thread, shape, dtype) -> pinned staging tensor of d2h(scratch=True), LRU, <= 64 entries
        self.h2d_bytes = 0      # bytes moved host->device / device->host through h2d()/d2h() (bench.py e2e accounting)
        self.d2h_bytes = 0

    def h2d(self, t, dtype=None) -> torch.Tensor:
        """Host array/tensor -> device tensor (async when the source is pinned); counts the bytes."""
        t = torch.as_tensor(t)
        if t.device.type == "cpu":
            self.h2d_bytes += t.numel() * t.element_size()
        t = t.to(self.device, non_blocking=True)
        return t if dtype is None else t.to(dtype)

    def d2h(self, t: torch.Tensor, scratch: bool = False) -> np.ndarray:
        """Device tensor -> numpy.  `scratch=True` (large tensors the caller consumes before ITS next d2h of the same shape,
        e.g. the detector's probability map) lands in a per-thread pinned buffer: the copy runs at full PCIe rate instead of
        staging through pageable memory while the page threads' kernels queue behind it on the shared stream.  The returned
        array is a view of that buffer - never hand it to the caller of the plugin."""
        with trace("d2h"):
            return self._d2h(t, scratch)

    def _d2h(self, t: torch.Tensor, scratch: bool = False) -> np.ndarray:
        self.d2h_bytes += t.numel() * t.element_size()
        if scratch and self._pinned is not None and t.is_cuda and t.numel() * t.element_size() >= (1 << 20):
            key = (threading.get_ident(), tuple(t.shape), t.dtype)
            with self._pin_lock:
                buf = self._pinned.get(key)
                if buf is not None:
                    self._pinned.move_to_end(key)
            if buf is None:
                try:
                    buf = torch.empty(tuple(t.shape), dtype=t.dtype, pin_memory=True)
                except RuntimeError:                      # the host cannot pin more memory: pageable copies from now on
                    self._pinned = None
                    return t.cpu().numpy()
                with self._pin_lock:
                    self._pinned[key] = buf
                    while len(self._pinned) > 64:         # page sizes / worker threads changed: drop the least recently used buffer
                        self._pinned.popitem(last=False)
            buf.copy_(t, non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            return buf.numpy()
        return t.cpu().numpy()

    # ------------------------------------------------------------------ plumbing
    def close(self):
        if getattr(self, "_h", None):
            self.lib.mitb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise MitbError(self.lib.mitb_last_error(self._h).decode())

    def _call(self, fn, *args):
        with trace("enqueue(lock+launch)"):
            with self._lock:
                self._check(fn(self._h, *args))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_tensor_cores(self, on: bool):
        """Process-wide: route eligible convolutions to the tcgen05 kernel (default) or keep everything on the fp32 SIMT kernel."""
        with self._lock:
            self.lib.mitb_set_tensor_cores(1 if on else 0)

    def set_sparse_decoder(self, on: bool):
        """Process-wide: output-sparse LaMa decoder (default on); off = every tile of the upsampling stages is computed."""
        with self._lock:
            self.lib.mitb_set_sparse_decoder(1 if on else 0)

    def set_ffc_mode(self, mode: int):
        """Process-wide LaMa FFC implementation: 0 generic planar, 1 fused NHWC when no layer needs split-K (default), 2 fused whenever capable."""
        with self._lock:
            self.lib.mitb_set_ffc_mode(int(mode))

    def profile(self, on: bool):
        self._call(self.lib.mitb_profile_enable, 1 if on else 0)

    def profile_report(self) -> dict:
        import json
        with self._lock:
            return json.loads(self.lib.mitb_profile_report(self._h).decode())

    @property
    def launches(self) -> int:
        return int(self.lib.mitb_launch_count(self._h))

    @property
    def workspace_bytes(self) -> int:
        return int(self.lib.mitb_workspace_bytes(self._h))

    def _tensors(self, sd: Dict[str, torch.Tensor]):
        keep, arr = [], (MitbTensor * len(sd))()
        for i, (k, v) in enumerate(sd.items()):
            t = v.detach().to(device=self.device, dtype=torch.float32).contiguous()
            keep.append(t)
            arr[i].name = k.encode()
            arr[i].data = t.data_ptr()
            arr[i].ndim = t.dim()
            for d in range(t.dim()):
                arr[i].shape[d] = t.shape[d]
        return arr, keep

    @staticmethod
    def _float_sd(sd):
        return {k: v for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point() and v.dim() <= 4}

    # ------------------------------------------------------------------ models
    def load_dbnet(self, state_dict):
        arr, keep = self._tensors(self._float_sd(state_dict))
        self._call(self.lib.mitb_dbnet_load, arr, len(arr))
        torch.cuda.synchronize(self.device)

    def unload_dbnet(self):
        with self._lock:          # never free a model while another thread is enqueueing its forward
            self._check(self.lib.mitb_dbnet_unload(self._h))

    def dbnet_forward(self, x: torch.Tensor):
        """x: float32 [n,3,h,w] normalised, or uint8 [n,h,w,3]; returns (db sigmoid [n,2,h,w], mask [n,1,h/2,w/2])."""
        x = x.to(self.device).contiguous()
        if x.dtype == torch.uint8:
            n, h, w, _ = x.shape
        else:
            n, _, h, w = x.shape
        db = torch.empty((n, 2, h, w), dtype=torch.float32, device=self.device)
        mask = torch.empty((n, 1, h // 2, w // 2), dtype=torch.float32, device=self.device)
        fn = self.lib.mitb_dbnet_forward_u8 if x.dtype == torch.uint8 else self.lib.mitb_dbnet_forward
        self._call(fn, _ptr(x), n, h, w, _ptr(db), _ptr(mask), self._stream())
        return db, mask

    def load_dbnet_r34(self, state_dict):
        """The default detector's network (TextDetection, DBNet_resnet34.py); its own slot next to load_dbnet's."""
        arr, keep = self._tensors(self._float_sd(state_dict))
        self._call(self.lib.mitb_dbnet_r34_load, arr, len(arr))
        torch.cuda.synchronize(self.device)

    def unload_dbnet_r34(self):
        with self._lock:          # never free a model while another thread is enqueueing its forward
            self._check(self.lib.mitb_dbnet_r34_unload(self._h))

    def dbnet_r34_forward(self, x: torch.Tensor):
        """x: float32 [n,3,h,w] normalised, or uint8 [n,h,w,3], h and w multiples of 256; returns (db sigmoid [n,2,h,w], mask [n,1,h/2,w/2])."""
        x = x.to(self.device).contiguous()
        if x.dtype == torch.uint8:
            n, h, w, _ = x.shape
        else:
            n, _, h, w = x.shape
        db = torch.empty((n, 2, h, w), dtype=torch.float32, device=self.device)
        mask = torch.empty((n, 1, h // 2, w // 2), dtype=torch.float32, device=self.device)
        fn = self.lib.mitb_dbnet_r34_forward_u8 if x.dtype == torch.uint8 else self.lib.mitb_dbnet_r34_forward
        self._call(fn, _ptr(x), n, h, w, _ptr(db), _ptr(mask), self._stream())
        return db, mask

    def load_ocr(self, state_dict, pe_table: Optional[torch.Tensor] = None):
        sd = self._float_sd(state_dict)
        sd = {k: v for k, v in sd.items() if not k.endswith("pe.pe")}
        if pe_table is not None:
            sd["pe.table"] = pe_table
        arr, keep = self._tensors(sd)
        self._call(self.lib.mitb_ocr_load, arr, len(arr))
        torch.cuda.synchronize(self.device)

    def unload_ocr(self):
        with self._lock:          # never free a model while another thread is enqueueing its forward
            self._check(self.lib.mitb_ocr_unload(self._h))

    def ocr_forward(self, x: torch.Tensor):
        """x: float32 [n,3,48,wp] normalised or uint8 [n,48,wp,3]; returns (argmax int32 [n,T], logprob [n,T], colors [n,T,6])."""
        x = x.to(self.device).contiguous()
        if x.dtype == torch.uint8:
            n, _, wp, _ = x.shape
        else:
            n, _, _, wp = x.shape
        T = self.lib.mitb_ocr_timesteps(wp)
        idx = torch.empty((n, T), dtype=torch.int32, device=self.device)
        lp = torch.empty((n, T), dtype=torch.float32, device=self.device)
        col = torch.empty((n, T, 6), dtype=torch.float32, device=self.device)
        fn = self.lib.mitb_ocr_forward_u8 if x.dtype == torch.uint8 else self.lib.mitb_ocr_forward
        self._call(fn, _ptr(x), n, wp, _ptr(idx), _ptr(lp), _ptr(col), self._stream())
        return idx, lp, col

    def load_lama(self, gen_state_dict, mpe_state_dict=None):
        sd = self._float_sd(gen_state_dict)
        if mpe_state_dict is not None:
            for k, v in mpe_state_dict.items():
                sd["mpe." + k] = v
        arr, keep = self._tensors(sd)
        self._call(self.lib.mitb_lama_load, arr, len(arr))
        torch.cuda.synchronize(self.device)

    def unload_lama(self):
        with self._lock:          # never free a model while another thread is enqueueing its forward
            self._check(self.lib.mitb_lama_unload(self._h))

    def lama_forward(self, img: torch.Tensor, mask: torch.Tensor, rel_pos=None, direct=None, tables256=False):
        """rel_pos/direct: full-resolution MPE tables [n,h,w]/[n,h,w,4], or (tables256=True) the 256x256 ones."""
        img = img.to(self.device, torch.float32).contiguous()
        mask = mask.to(self.device, torch.float32).contiguous()
        n, _, h, w = img.shape
        if rel_pos is not None:
            rel_pos = torch.as_tensor(rel_pos).to(self.device, torch.int32).contiguous()
            direct = torch.as_tensor(direct).to(self.device, torch.int32).contiguous()
        out = torch.empty_like(img)
        fn = self.lib.mitb_lama_forward_mpe256 if (tables256 and rel_pos is not None) else self.lib.mitb_lama_forward
        self._call(fn, _ptr(img), _ptr(mask), _ptr(rel_pos), _ptr(direct), n, h, w, _ptr(out), self._stream())
        return out

    def lama_infer_u8(self, img_u8: torch.Tensor, mask_u8: torch.Tensor, rel256=None, direct256=None, composite=True):
        """Device part of LamaMPEInpainter._infer on uint8 data: img [h,w,3], mask [h,w] (device, network resolution)."""
        h, w, _ = img_u8.shape
        out = torch.empty_like(img_u8)
        self._call(self.lib.mitb_lama_infer_u8, _ptr(img_u8), _ptr(mask_u8), _ptr(rel256), _ptr(direct256), h, w,
                                                1 if composite else 0, _ptr(out), self._stream())
        return out

    # ------------------------------------------------------------------ standalone operators (tests / micro-benchmarks)
    def _dev(self, t, dtype=torch.float32):
        return None if t is None else torch.as_tensor(t).to(self.device, dtype).contiguous()

    def conv2d(self, x, w, bias=None, stride=(1, 1), padding=(0, 0), pad_mode="zeros", act=0, in_scale=None, in_shift=None,
               in_relu=False):
        x, w, bias, in_scale, in_shift = map(self._dev, (x, w, bias, in_scale, in_shift))
        n, cin, h, wd = x.shape
        cout, _, kh, kw = w.shape
        ho = (h + 2 * padding[0] - kh) // stride[0] + 1
        wo = (wd + 2 * padding[1] - kw) // stride[1] + 1
        y = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_conv2d, _ptr(x), n, cin, h, wd, _ptr(w), cout, kh, kw, stride[0], stride[1],
                                            padding[0], padding[1], 1 if pad_mode == "reflect" else 0, _ptr(bias), act,
                                            _ptr(in_scale), _ptr(in_shift), int(in_relu), _ptr(y), self._stream())
        return y

    def conv_transpose2d(self, x, w, bias=None, k=2, pad=0, out_pad=0, act=0):
        x, w, bias = map(self._dev, (x, w, bias))
        n, cin, h, wd = x.shape
        cout = w.shape[1]
        y = torch.empty((n, cout, 2 * h, 2 * wd), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_conv_transpose2d, _ptr(x), n, cin, h, wd, _ptr(w), cout, k, pad, out_pad,
                                                      _ptr(bias), act, _ptr(y), self._stream())
        return y

    def dwconv7_ln(self, x, wdw, bdw, lnw, lnb, eps=1e-6):
        x, wdw, bdw, lnw, lnb = map(self._dev, (x, wdw, bdw, lnw, lnb))
        n, c, h, w = x.shape
        y = torch.empty_like(x)
        self._call(self.lib.mitb_op_dwconv7_ln, _ptr(x), n, c, h, w, _ptr(wdw), _ptr(bdw), _ptr(lnw), _ptr(lnb),
                                                eps, _ptr(y), self._stream())
        return y

    def maxpool3x3s2(self, x):
        """F.max_pool2d(x, 3, 2, 1) of an NCHW float32 tensor (exact)."""
        x = self._dev(x)
        n, c, h, w = x.shape
        y = torch.empty((n, c, (h - 1) // 2 + 1, (w - 1) // 2 + 1), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_maxpool3x3s2, _ptr(x), n, c, h, w, _ptr(y), self._stream())
        return y

    def layernorm(self, x, w, b, eps):
        x, w, b = map(self._dev, (x, w, b))
        rows, c = x.shape
        y = torch.empty_like(x)
        self._call(self.lib.mitb_op_layernorm, _ptr(x), rows, c, _ptr(w), _ptr(b), eps, _ptr(y), self._stream())
        return y

    def rfft2(self, x):
        x = self._dev(x)
        c, h, w = x.shape
        spec = torch.empty((2 * c, h, w // 2 + 1), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_rfft2, _ptr(x), c, h, w, _ptr(spec), self._stream())
        return spec

    def irfft2(self, spec, w):
        spec = self._dev(spec)
        c2, h, _ = spec.shape
        y = torch.empty((c2 // 2, h, w), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_irfft2, _ptr(spec), c2 // 2, h, w, _ptr(y), self._stream())
        return y

    def rfft2_nhwc(self, x):
        x = self._dev(x)
        n, h, w, c = x.shape
        spec = torch.empty((n, h, w // 2 + 1, 2 * c), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_rfft2_nhwc, _ptr(x), n, h, w, c, _ptr(spec), self._stream())
        return spec

    def irfft2_nhwc(self, spec, w, add=None):
        spec, add = self._dev(spec), self._dev(add)
        n, h, _, c2 = spec.shape
        y = torch.empty((n, h, w, c2 // 2), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_irfft2_nhwc, _ptr(spec), _ptr(add), n, h, w, c2 // 2, _ptr(y), self._stream())
        return y

    def attention(self, qk, v, n, t, heads, hd):
        qk, v = map(self._dev, (qk, v))
        out = torch.empty_like(v)
        self._call(self.lib.mitb_op_attention, _ptr(qk), _ptr(v), n, t, heads, hd, _ptr(out), self._stream())
        return out

    def mpe_tables_256(self, small_u8):
        """Device version of host.mpe._tables_256: INTER_AREA-reduced uint8 mask [256,256] (or [n,256,256]) -> (rel_pos, direct) int32."""
        s = torch.as_tensor(small_u8)
        if s.device.type == "cpu":
            s = self.h2d(s)
        s = s.to(torch.uint8).contiguous()
        n = 1 if s.dim() == 2 else s.shape[0]
        rel = torch.empty((n, 256, 256), dtype=torch.int32, device=self.device)
        direct = torch.empty((n, 256, 256, 4), dtype=torch.int32, device=self.device)
        self._call(self.lib.mitb_op_mpe_tables, _ptr(s), n, _ptr(rel), _ptr(direct), self._stream())
        return rel, direct

    def bilateral17(self, img_u8):
        img = torch.as_tensor(img_u8).to(self.device, torch.uint8).contiguous()
        h, w, _ = img.shape
        out = torch.empty_like(img)
        self._call(self.lib.mitb_op_bilateral17, _ptr(img), h, w, _ptr(out), self._stream())
        return out

    def warp_lines(self, page: torch.Tensor, records: np.ndarray, canvas_w: int, canvas_h: int = 48) -> torch.Tensor:
        """Perspective crops of the text lines of one OCR chunk straight into the chunk canvas (row O3 on the device).
        page: uint8 [H,W,3] CUDA tensor; records: float64 [n,16] from host.geometry.warp_record; returns uint8 [n,canvas_h,canvas_w,3]."""
        assert page.is_cuda and page.dtype == torch.uint8 and page.dim() == 3 and page.shape[2] == 3 and page.is_contiguous()
        if isinstance(records, torch.Tensor) and records.is_cuda:
            rec = records.contiguous()
            assert rec.dtype == torch.float64
        else:
            rec = self.h2d(np.ascontiguousarray(records, dtype=np.float64))
        assert rec.dim() == 2 and rec.shape[1] == 16
        n = int(rec.shape[0])
        canvas = torch.empty((n, canvas_h, canvas_w, 3), dtype=torch.uint8, device=self.device)
        self._call(self.lib.mitb_op_warp_lines_u8, _ptr(page), int(page.shape[0]), int(page.shape[1]), _ptr(rec), n, _ptr(canvas), canvas_h,
                   canvas_w, self._stream())
        return canvas

    def textline_pairs(self, features: np.ndarray, params) -> np.ndarray:
        """`can_merge_region` for every pair of lines (SURVEY 8f N3): features float64 [n,16] (host.geometry.pair_features), params =
        (ratio, discard_connection_gap, char_gap_tolerance, char_gap_tolerance2, font_size_ratio_tol, aspect_ratio_tol); returns uint8
        [n,n] on the host (1 mergeable, 0 not, 2 undecided)."""
        f = self.h2d(np.ascontiguousarray(features, dtype=np.float64))
        n = int(f.shape[0])
        adj = torch.empty((n, n), dtype=torch.uint8, device=self.device)
        self._call(self.lib.mitb_op_textline_pairs, _ptr(f), n, *[C.c_double(float(v)) for v in params], _ptr(adj), self._stream())
        return self.d2h(adj).copy()

    def ctc_collapse(self, idx: torch.Tensor, logprob: torch.Tensor, colors: torch.Tensor):
        """Greedy CTC collapse on the device (row O8): returns (counts [n], steps [n,T], chars [n,T], logprob [n,T], colors [n,T,6]) with
        the kept steps compacted to the front of each row; entries past counts[i] are unspecified."""
        n, T = idx.shape
        counts = torch.empty((n,), dtype=torch.int32, device=self.device)
        steps = torch.empty((n, T), dtype=torch.int32, device=self.device)
        chars = torch.empty((n, T), dtype=torch.int32, device=self.device)
        lp = torch.empty((n, T), dtype=torch.float32, device=self.device)
        col = torch.empty((n, T, 6), dtype=torch.float32, device=self.device)
        self._call(self.lib.mitb_op_ctc_collapse, _ptr(idx.contiguous()), _ptr(logprob.contiguous()), _ptr(colors.contiguous()), n, T,
                   _ptr(counts), _ptr(steps), _ptr(chars), _ptr(lp), _ptr(col), self._stream())
        return counts, steps, chars, lp, col


_engines = {}


def get_engine(device="cuda:0") -> Engine:
    """Process-wide engine per device (the three plugins of one process share workspace and stream)."""
    key = str(torch.device(device if str(device) != "cuda" else "cuda:0"))
    if key not in _engines:
        _engines[key] = Engine(key)
    return _engines[key]

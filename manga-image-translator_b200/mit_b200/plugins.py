"""Drop-in plugin classes for the three dense-inference stages, same names / signatures / return types as the reference:

  DBConvNextDetector   manga_translator/detection/dbnet_convnext.py:512-588
  DefaultDetector      manga_translator/detection/default.py:27-103 (DBNet-ResNet34; same host glue as DBConvNextDetector)
  Model48pxCTCOCR      manga_translator/ocr/model_48px_ctc.py:18-160
  LamaMPEInpainter     manga_translator/inpainting/inpainting_lama_mpe.py:26-118
  LamaLargeInpainter   manga_translator/inpainting/inpainting_lama_mpe.py:121-136

``register()`` swaps them into the reference registries (detection/__init__.py:12-20, ocr/__init__.py:11-18,
inpainting/__init__.py:13-22).  All tensor math runs in libmitb (hand-written CUDA through the C ABI); torch tensors are
device-memory containers only.  CUDA only: any other device string raises (no CPU fallback).

Weights: the same checkpoint files and key layouts as the reference (``sd['model']``|``sd``; ``gen_state_dict`` +
``str_state_dict``).  Because no checkpoint is downloadable offline, tests and the bench may inject a state_dict with
``Plugin.set_state_dict(...)`` instead of writing a file.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional

import cv2
import numpy as np
import torch

from . import compat
from .compat import InpainterConfig, OcrConfig, OfflineDetector, OfflineInpainter, OfflineOCR, Quadrilateral, chunks
from .engine import Engine, get_engine, trace
from ._lib import MitbError
from .host import det_post, mpe, rearrange
from .host.geometry import warp_record


def _require_cuda(device: str) -> str:
    if not str(device).startswith("cuda"):
        raise MitbError(f"mit_b200 plugins run on CUDA (H100) only; got device '{device}'. "
                        f"Use the reference classes for CPU execution.")
    return "cuda:0" if device == "cuda" else device


class _InjectableWeights:
    _injected: Optional[dict] = None

    @classmethod
    def set_state_dict(cls, sd: Optional[dict]):
        """Use an in-memory state_dict instead of the checkpoint file (tests / bench; pass None to reset)."""
        cls._injected = sd


# ----------------------------------------------------------------------------------------------- detector
class DBConvNextDetector(_InjectableWeights, OfflineDetector):
    # The reference mapping carries an empty URL, which its own ModelWrapper rejects (SURVEY F6): file-only here.
    _MODEL_MAPPING = {}
    _CKPT = "dbnet_convnext.ckpt"

    async def _load(self, device: str):
        self.device = _require_cuda(device)
        self.engine: Engine = get_engine(self.device)
        sd = self._injected
        if sd is None:
            sd = torch.load(self._get_file_path(self._CKPT), map_location="cpu")
        self._load_net(sd["model"] if "model" in sd else sd)

    async def _unload(self):
        self._unload_net()

    # the network behind the shared `_infer` glue: one hook to load it, one to unload it, one to run a device batch
    def _load_net(self, sd):
        self.engine.load_dbnet(sd)

    def _unload_net(self):
        self.engine.unload_dbnet()

    def _net_forward(self, batch):
        return self.engine.dbnet_forward(batch)

    def _batch_forward(self, batch_u8: np.ndarray):
        """det_batch_forward_default (dbnet_convnext.py:499-509) on uint8 NHWC: normalise + forward + sigmoid on device."""
        db, mask = self._net_forward(self.engine.h2d(np.ascontiguousarray(batch_u8)))
        return self.engine.d2h(db), self.engine.d2h(mask)

    async def _infer(self, image: np.ndarray, detect_size: int, text_threshold: float, box_threshold: float,
                     unclip_ratio: float, verbose: bool = False):
        eng = self.engine
        db, mask = rearrange.rearrange_forward(image, self._batch_forward, detect_size, 4)
        if db is None:
            # cv2.bilateralFilter(image, 17, 80, 80) on the GPU (dbnet_convnext.py:549)
            img_dev = eng.h2d(np.ascontiguousarray(image))
            filt = eng.bilateral17(img_dev)
            h, w = image.shape[:2]
            ratio = detect_size / max(h, w)
            th, tw = int(round(h * ratio)), int(round(w * ratio))
            if (th, tw) == (h, w) and th % 256 == 0 and tw % 256 == 0:
                batch, pad_w, pad_h, target_ratio = filt[None], 0, 0, ratio     # stays on the device
                rh, rw = h, w
            else:
                resized, target_ratio, _, pad_w, pad_h = det_post.resize_aspect_ratio(eng.d2h(filt), detect_size,
                                                                                       cv2.INTER_LINEAR, mag_ratio=1)
                rh, rw = resized.shape[:2]
                batch = eng.h2d(resized[None])
            ratio_h = ratio_w = 1 / target_ratio
            db_t, mask_t = self._net_forward(batch)
            db, mask = eng.d2h(db_t[:, :1].contiguous(), scratch=True), eng.d2h(mask_t, scratch=True)   # consumed below, never returned
            img_resized_h, img_resized_w = rh, rw
        else:
            img_resized_h, img_resized_w = image.shape[:2]
            ratio_w = ratio_h = 1
            pad_h = pad_w = 0
        self.logger.info(f"Detection resolution: {img_resized_w}x{img_resized_h}")

        mask = mask[0, 0, :, :]
        with trace("host:det_post"):
            boxes, scores = det_post.boxes_from_prob(db[0, 0], text_threshold, box_threshold, unclip_ratio, img_resized_w, img_resized_h)
            polys = det_post.polys_from_boxes(boxes, scores, ratio_w, ratio_h)
            textlines = [Quadrilateral(pts.astype(int), "", score) for pts, score in zip(polys, scores)]
            textlines = list(filter(lambda q: q.area > 16, textlines))
        with trace("host:det_mask"):
            mask_resized = cv2.resize(mask, (mask.shape[1] * 2, mask.shape[0] * 2), interpolation=cv2.INTER_LINEAR)
            if pad_h > 0:
                mask_resized = mask_resized[:-pad_h, :]
            elif pad_w > 0:
                mask_resized = mask_resized[:, :-pad_w]
            raw_mask = np.clip(mask_resized * 255, 0, 255).astype(np.uint8)
        return textlines, raw_mask, None


class DefaultDetector(DBConvNextDetector):
    """The reference's `default` detector: DBNet-ResNet34 (detection/default_utils/DBNet_resnet34.py).  Its `_infer`
    (default.py:56-103) is line for line DBConvNextDetector's, so only the network differs.  Unlike the reference constructor
    (default.py:36-40) it neither creates the model directory nor moves a checkpoint found in the working directory."""
    _MODEL_MAPPING = {
        'model': {
            'url': 'https://github.com/zyddnys/manga-image-translator/releases/download/beta-0.3/detect-20241225.ckpt',
            'hash': '67ce1c4ed4793860f038c71189ba9630a7756f7683b1ee5afb69ca0687dc502e',
            'file': '.',
        }
    }
    _CKPT = "detect-20241225.ckpt"
    _injected: Optional[dict] = None          # its own injected weights, not DBConvNextDetector's

    def _load_net(self, sd):
        self.engine.load_dbnet_r34(sd)

    def _unload_net(self):
        self.engine.unload_dbnet_r34()

    def _net_forward(self, batch):
        return self.engine.dbnet_r34_forward(batch)


# ----------------------------------------------------------------------------------------------- OCR
def _pe_table(max_len: int = 2048, d: int = 320) -> torch.Tensor:
    """PositionalEncoding buffer, computed with the same torch ops as the reference (model_48px_ctc.py:168-174) so the
    table is bit-identical to the one its modules hold."""
    pe = torch.zeros(max_len, d)
    position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d, 2).float() * (-math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def ctc_collapse(idx: np.ndarray, blank: int = 0):
    """Greedy CTC collapse over all timesteps (model_48px_ctc.py:464-493), vectorised: returns per line the kept timesteps."""
    prev = np.concatenate([np.full((idx.shape[0], 1), blank, idx.dtype), idx[:, :-1]], axis=1)
    keep = (idx != prev) & (idx != blank)
    return [np.nonzero(k)[0] for k in keep]


class Model48pxCTCOCR(_InjectableWeights, OfflineOCR):
    _MODEL_MAPPING = {}
    _CKPT = "ocr-ctc.ckpt"
    _DICT = "alphabet-all-v5.txt"
    _injected_dictionary: Optional[List[str]] = None

    @classmethod
    def set_dictionary(cls, dictionary: Optional[List[str]]):
        cls._injected_dictionary = dictionary

    async def _load(self, device: str):
        self.device = _require_cuda(device)
        self.engine: Engine = get_engine(self.device)
        if self._injected_dictionary is not None:
            self.dictionary = list(self._injected_dictionary)
        else:
            with open(self._get_file_path(self._DICT), "r", encoding="utf-8") as fp:
                self.dictionary = [s[:-1] for s in fp.readlines()]
        sd = self._injected
        if sd is None:
            sd = torch.load(self._get_file_path(self._CKPT), map_location="cpu")
        sd = sd["model"] if "model" in sd else sd
        sd = {k: v for k, v in sd.items() if not k.endswith(".pe.pe")}
        if sd["char_pred.weight"].shape[0] != len(self.dictionary):
            raise MitbError(f"dictionary has {len(self.dictionary)} entries, char_pred has {sd['char_pred.weight'].shape[0]}")
        self.engine.load_ocr(sd, _pe_table())

    async def _unload(self):
        self.engine.unload_ocr()

    def _generate_text_direction(self, bboxes):
        """CommonOCR._generate_text_direction (ocr/common.py:12-39) with the O(n^2) pair predicate on the device (SURVEY 8f N3);
        MITB_HOST_PAIRS=1 keeps the host evaluation."""
        from .host.geometry import generate_text_direction
        eng = None if os.environ.get("MITB_HOST_PAIRS", "0") == "1" else getattr(self, "engine", None)
        if eng is not None and not (hasattr(eng, "textline_pairs") and all(isinstance(b, Quadrilateral) for b in bboxes)):
            eng = None
        yield from generate_text_direction(bboxes, engine=eng)

    async def _infer(self, image: np.ndarray, textlines: List[Quadrilateral], config: OcrConfig, verbose: bool = False):
        text_height, max_chunk_size = 48, 16
        ignore_bubble = getattr(config, "ignore_bubble", 0)
        threshold = 0.5 if getattr(config, "prob", None) is None else config.prob
        with trace("host:ocr_direction"):
            quadrilaterals = list(self._generate_text_direction(textlines))
        # Crops: by default on the device (SURVEY 8f N2 / O3): the host solves the 4-point homographies, one kernel per chunk warps the
        # lines out of the resident page straight into the chunk canvas (bit-exact with cv2.warpPerspective + rotate).  The bubble
        # filter needs the crops on the host, so it keeps the reference's own sequence (MITB_HOST_CROPS=1 forces that path too).
        host_crops = ((1 <= ignore_bubble <= 50) or os.environ.get("MITB_HOST_CROPS", "0") == "1" or image.dtype != np.uint8 or image.ndim != 3
                      or image.shape[2] != 3 or not all(isinstance(q, Quadrilateral) for q, _ in quadrilaterals))
        eng = self.engine
        if host_crops:
            with trace("host:ocr_crops"):
                region_imgs = [q.get_transformed_region(image, d, text_height) for q, d in quadrilaterals]
            line_w = [r.shape[1] for r in region_imgs]
        else:
            with trace("host:ocr_homography"):
                recs = [warp_record(q, image.shape[0], image.shape[1], d, text_height) for q, d in quadrilaterals]
            line_w = [w for _, w in recs]
            rec_arr = np.stack([r for r, _ in recs]) if recs else np.zeros((0, 16), dtype=np.float64)
            page_dev = eng.h2d(np.ascontiguousarray(image)) if recs else None
        out_regions = []
        perm = range(len(line_w))
        is_quadrilaterals = False
        if len(quadrilaterals) > 0 and isinstance(quadrilaterals[0][0], Quadrilateral):
            is_quadrilaterals = True
            perm = sorted(range(len(line_w)), key=lambda x: line_w[x])
        if 1 <= ignore_bubble <= 50:
            from .host.bubble import is_ignore
        for indices in chunks(perm, max_chunk_size):
            N = len(indices)
            widths = [line_w[i] for i in indices]
            max_width = (4 * (max(widths) + 7) // 4) + 128
            if host_crops:
                region = np.zeros((N, text_height, max_width, 3), dtype=np.uint8)
                for i, idx in enumerate(indices):
                    if 1 <= ignore_bubble <= 50 and is_ignore(region_imgs[idx], ignore_bubble):
                        continue
                    region[i, :, :widths[i], :] = region_imgs[idx]
                region_dev = eng.h2d(region)
            else:
                region_dev = eng.warp_lines(page_dev, rec_arr[list(indices)], max_width, text_height)
            # (x-127.5)/127.5 normalisation, network, log-softmax/argmax, colour clamp and the greedy CTC collapse all run on the device
            pred, logprob, colors = eng.ocr_forward(region_dev)
            counts, _, kept_ch, kept_lp, kept_col = eng.ctc_collapse(pred, logprob, colors)
            counts, kept_ch, kept_lp, kept_col = eng.d2h(counts), eng.d2h(kept_ch), eng.d2h(kept_lp), eng.d2h(kept_col)
            for i in range(N):
                cnt = int(counts[i])
                if cnt == 0:
                    continue
                chars = [self.dictionary[c] for c in kept_ch[i, :cnt]]
                chars = [" " if ch == "<SP>" else ch for ch in chars]
                prob = np.exp(np.mean(kept_lp[i, :cnt].astype(np.float64)))           # mean of python floats == float64 mean
                if prob < threshold:
                    continue
                txt = "".join(chars)
                sel = [k for k, ch in enumerate(chars) if ch != " "]
                cols = [0] * 6
                if sel:
                    ints = (kept_col[i, sel].astype(np.float64) * 255).astype(np.int64)  # int(float(v) * 255) per element
                    cols = [int(ints[:, k].sum() / len(sel)) for k in range(6)]
                fr, fg, fb, br, bg, bb = cols
                self.logger.info(f"prob: {prob} {txt} fg: ({fr}, {fg}, {fb}) bg: ({br}, {bg}, {bb})")
                cur_region = quadrilaterals[indices[i]][0]
                if isinstance(cur_region, Quadrilateral):
                    cur_region.text = txt
                    cur_region.prob = prob
                    cur_region.fg_r, cur_region.fg_g, cur_region.fg_b = fr, fg, fb
                    cur_region.bg_r, cur_region.bg_g, cur_region.bg_b = br, bg, bb
                else:
                    cur_region.text.append(txt)
                    cur_region.update_font_colors(np.array([fr, fg, fb]), np.array([br, bg, bb]))
                out_regions.append(cur_region)
        if is_quadrilaterals:
            return out_regions
        return textlines


# ----------------------------------------------------------------------------------------------- inpainter
class LamaMPEInpainter(_InjectableWeights, OfflineInpainter):
    _MODEL_MAPPING = {}
    _CKPT = "inpainting_lama_mpe.ckpt"
    _USE_MPE = True

    async def _load(self, device: str):
        self.device = _require_cuda(device)
        self.engine: Engine = get_engine(self.device)
        sd = self._injected
        if sd is None:
            sd = torch.load(self._get_file_path(self._CKPT), map_location="cpu")
        self.engine.load_lama(sd["gen_state_dict"], sd["str_state_dict"] if self._USE_MPE else None)

    async def _unload(self):
        self.engine.unload_lama()

    async def _infer(self, image: np.ndarray, mask: np.ndarray, config: InpainterConfig, inpainting_size: int = 1024,
                     verbose: bool = False, _device_out: bool = False) -> np.ndarray:
        """`_device_out` (not part of the reference signature; used by the multi-GPU driver): when the page needed no host-side
        resize, return the composited uint8 page as a CUDA tensor instead of copying it to the host."""
        if image.dtype != np.uint8 or mask.dtype != np.uint8:
            raise MitbError(f"inpainter expects uint8 image and mask (got {image.dtype}, {mask.dtype}), like the reference pipeline passes")
        img_original, mask_full = image, mask          # inputs are borrowed: never written; the host composite below (only taken
        height, width, _ = image.shape                 # when the page had to be resized) derives its own {0,1} mask from them
        if max(image.shape[0:2]) > inpainting_size:
            r = float(inpainting_size) / max(image.shape[0], image.shape[1])
            size = (round(image.shape[1] * r), round(image.shape[0] * r))
            image = cv2.resize(image, size, interpolation=cv2.INTER_LINEAR_EXACT)
            mask = cv2.resize(mask, size, interpolation=cv2.INTER_LINEAR_EXACT)
        h, w, _ = image.shape
        new_h = h if h % 8 == 0 else h + (8 - h % 8)
        new_w = w if w % 8 == 0 else w + (8 - w % 8)
        if new_h != h or new_w != w:
            image = cv2.resize(image, (new_w, new_h), interpolation=cv2.INTER_LINEAR)
            mask = cv2.resize(mask, (new_w, new_h), interpolation=cv2.INTER_LINEAR)
        self.logger.info(f"Inpainting resolution: {new_w}x{new_h}")
        eng = self.engine
        resized = (new_h, new_w) != (height, width)
        rel_pos = direct = None
        if self._USE_MPE:
            # 256x256 tables on the host (binary morphology on a tiny image); upsampled inside the kernel
            if mask.dtype == np.uint8:
                mask01 = mask >= 128                   # == (mask / 255 >= 0.5) for uint8: 127/255 < 0.5 <= 128/255
            else:
                mask01 = ((mask.astype(np.float32) / 255.0) >= 0.5).astype(np.float32)
            # 256x256 INTER_AREA reduction on the host (cv2 defines it), the iterative distance / direction sweep on the device
            with trace("host:mpe_small"):
                small = mpe.small_mask_256(mask01)
            rel_pos, direct = eng.mpe_tables_256(small)
        # /255, mask binarisation, pre-masking, network, blend, (x*255) truncation and (when no resize happened) the final
        # composite with the original page all run on the device; only uint8 crosses the bus.
        out_dev = eng.lama_infer_u8(eng.h2d(np.ascontiguousarray(image)), eng.h2d(np.ascontiguousarray(mask)), rel_pos, direct,
                                    composite=not resized)
        if _device_out and not resized:
            return out_dev
        img_inpainted = eng.d2h(out_dev, scratch=True).copy()      # pinned staging for the bus, then an owned array for the caller
        if not resized:
            return img_inpainted
        if new_h != height or new_w != width:
            img_inpainted = cv2.resize(img_inpainted, (width, height), interpolation=cv2.INTER_LINEAR)
        mask_original = (mask_full >= 127).astype(mask_full.dtype)[:, :, None]        # inpainting_lama_mpe.py:59-60
        return img_inpainted * mask_original + img_original * (1 - mask_original)


class LamaLargeInpainter(LamaMPEInpainter):
    _CKPT = "lama_large_512px.ckpt"
    _USE_MPE = False


# ----------------------------------------------------------------------------------------------- registration
def register(mask_refinement: bool = False, default_detector: bool = False):
    """Replace the reference registry entries with the H100 plugins (needs the real manga_translator package).  With
    `mask_refinement=True` also rebind `manga_translator.manga_translator.dispatch_mask_refinement` (manga_translator.py:34, called at
    :1356-1358) to the GPU stage of `mit_b200.mask_refinement` - same signature.  With `default_detector=True` also replace the
    reference's `default` detector (DBNet-ResNet34) with DefaultDetector."""
    if not compat.HAVE_REFERENCE:
        raise MitbError("register() needs an importable manga_translator package; see INTEGRATION.md")
    from manga_translator import detection, inpainting, ocr  # type: ignore
    from manga_translator.config import Detector, Inpainter, Ocr  # type: ignore
    detection.DETECTORS[Detector.dbconvnext] = DBConvNextDetector
    ocr.OCRS[Ocr.ocr48px_ctc] = Model48pxCTCOCR
    inpainting.INPAINTERS[Inpainter.lama_mpe] = LamaMPEInpainter
    inpainting.INPAINTERS[Inpainter.lama_large] = LamaLargeInpainter
    detection.detector_cache.pop(Detector.dbconvnext, None)
    ocr.ocr_cache.pop(Ocr.ocr48px_ctc, None)
    inpainting.inpainter_cache.pop(Inpainter.lama_mpe, None)
    inpainting.inpainter_cache.pop(Inpainter.lama_large, None)
    if default_detector:
        detection.DETECTORS[Detector.default] = DefaultDetector
        detection.detector_cache.pop(Detector.default, None)
    if mask_refinement:
        import manga_translator.manga_translator as mt  # type: ignore
        from . import mask_refinement as mr
        mt.dispatch_mask_refinement = mr.dispatch

"""Binding to the reference's plugin interface.

When ``manga_translator`` is importable (a real deployment) the plugin classes derive from ITS ``OfflineDetector`` /
``OfflineOCR`` / ``OfflineInpainter`` and use ITS ``Quadrilateral`` / config classes, so ``register()`` can drop them
into the reference registries unchanged.  When it is not (this repository's tests and bench: the package needs a dozen
third-party modules that are not installed) local stand-ins with the same names, signatures and lifecycle are used:

  InfererModule / ModelWrapper     manga_translator/utils/inference.py:24-27, 62-364 (load/unload/infer guards)
  OfflineDetector / CommonDetector manga_translator/detection/common.py:10-146
  OfflineOCR / CommonOCR           manga_translator/ocr/common.py:11-61
  OfflineInpainter                 manga_translator/inpainting/common.py:7-24
  OcrConfig / InpainterConfig      manga_translator/config.py:293-319 (only the fields the hot path reads)
"""
from __future__ import annotations

import logging
import os
from abc import ABC, abstractmethod
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

try:  # pragma: no cover - exercised only where the full reference package is installed
    from manga_translator.utils import InfererModule, ModelWrapper, Quadrilateral  # type: ignore
    from manga_translator.detection.common import OfflineDetector  # type: ignore
    from manga_translator.ocr.common import OfflineOCR  # type: ignore
    from manga_translator.inpainting.common import OfflineInpainter  # type: ignore
    from manga_translator.config import OcrConfig, InpainterConfig  # type: ignore
    HAVE_REFERENCE = True
except Exception:  # noqa: BLE001
    HAVE_REFERENCE = False
    from .host.geometry import Quadrilateral, generate_text_direction

    class InfererModule(ABC):
        def __init__(self):
            self.logger = logging.getLogger(self.__class__.__name__)
            super().__init__()

    class ModelWrapper(ABC):
        """Lifecycle of utils/inference.py:62-364 minus downloading (there is no network): files must already be in
        ``model_dir``; ``infer`` before ``load`` raises like the reference (:349-350)."""
        _MODEL_DIR = os.environ.get("MITB_MODEL_DIR", os.path.join(os.getcwd(), "models"))
        _MODEL_SUB_DIR = ""
        _MODEL_MAPPING = {}
        _KEY = ""

        def __init__(self):
            # nothing is downloaded, so no directory is created (the working directory may be read-only)
            self._key = self._KEY or self.__class__.__name__
            self._loaded = False

        @property
        def model_dir(self):
            return os.path.join(self._MODEL_DIR, self._MODEL_SUB_DIR)

        def _get_file_path(self, *args) -> str:
            return os.path.join(self.model_dir, *args)

        def is_loaded(self) -> bool:
            return self._loaded

        def is_downloaded(self) -> bool:
            return True

        async def download(self, force=False):
            return None

        async def reload(self, device: str, *args, **kwargs):
            await self.unload()
            await self.load(*args, **kwargs, device=device)

        async def load(self, device: str, *args, **kwargs):
            if not self.is_loaded():
                await self._load(*args, **kwargs, device=device)
                self._loaded = True

        async def unload(self):
            if self.is_loaded():
                await self._unload()
                self._loaded = False

        async def infer(self, *args, **kwargs):
            if not self.is_loaded():
                raise Exception(f"{self._key}: Tried to forward pass without having loaded the model.")
            return await self._infer(*args, **kwargs)

        @abstractmethod
        async def _load(self, device: str, *args, **kwargs):
            ...

        @abstractmethod
        async def _unload(self):
            ...

        @abstractmethod
        async def _infer(self, *args, **kwargs):
            ...

    class OfflineDetector(InfererModule, ModelWrapper):
        _MODEL_SUB_DIR = "detection"

        def __init__(self):
            InfererModule.__init__(self)
            ModelWrapper.__init__(self)

        async def detect(self, image: np.ndarray, detect_size: int, text_threshold: float, box_threshold: float,
                         unclip_ratio: float, invert: bool = False, gamma_correct: bool = False, rotate: bool = False,
                         auto_rotate: bool = False, verbose: bool = False):
            """CommonDetector.detect (detection/common.py:12-64): optional input variants around `_detect`, undone on the results.
            Order as in the reference: rotate 90 deg clockwise, zero border to a >= 400 px square when the short side is < 400,
            invert, gamma; then filter area > 1, crop the border, (auto_rotate: rerun rotated when most lines are horizontal),
            rotate the results back."""
            import cv2
            from collections import Counter
            page_h, page_w = image.shape[:2]
            original = image.copy()
            bordered = min(page_w, page_h) < 400
            work = image
            if rotate:
                work = np.rot90(work, k=-1)
            if bordered:
                side = max(work.shape[1], work.shape[0], 400)
                canvas = np.zeros((side, side, 3), np.uint8)
                canvas[:work.shape[0], :work.shape[1]] = work
                work = canvas
            if invert:
                work = cv2.bitwise_not(work)
            if gamma_correct:
                mean = np.mean(cv2.cvtColor(work, cv2.COLOR_BGR2GRAY))
                work = np.power(work, np.log(0.5 * 255) / np.log(mean)).clip(0, 255).astype(np.uint8)
            textlines, raw_mask, mask = await self._detect(work, detect_size, text_threshold, box_threshold, unclip_ratio, verbose)
            textlines = [t for t in textlines if t.area > 1]
            if bordered:
                bh, bw = work.shape[:2]
                raw_mask = cv2.resize(raw_mask, (bw, bh), interpolation=cv2.INTER_LINEAR)[:page_h, :page_w]
                if mask is not None:
                    mask = cv2.resize(mask, (bw, bh), interpolation=cv2.INTER_LINEAR)[:page_h, :page_w]
                kept = []
                for t in textlines:
                    if t.xyxy[0] >= page_w and t.xyxy[1] >= page_h:        # entirely inside the added border
                        continue
                    pts = t.pts
                    pts[:, 0] = np.clip(pts[:, 0], 0, page_w)
                    pts[:, 1] = np.clip(pts[:, 1], 0, page_h)
                    kept.append(Quadrilateral(pts, t.text, t.prob))
                textlines = kept
            if auto_rotate:
                votes = Counter("h" if t.aspect_ratio > 1 else "v" for t in textlines)
                if not textlines or votes.most_common(1)[0][0] == "h":
                    return await self.detect(original, detect_size, text_threshold, box_threshold, unclip_ratio, invert, gamma_correct,
                                             rotate=(not rotate), auto_rotate=False, verbose=verbose)
            if rotate:
                raw_mask = np.ascontiguousarray(np.rot90(raw_mask))
                if mask is not None:
                    mask = np.ascontiguousarray(np.rot90(mask).astype(np.uint8))
                back = []
                for t in textlines:
                    p = t.pts[:, [1, 0]]
                    p[:, 1] = page_h - p[:, 1]
                    back.append(Quadrilateral(p, t.text, t.prob))
                textlines = back
            return textlines, raw_mask, mask

        async def _detect(self, *args, **kwargs):
            return await self.infer(*args, **kwargs)

    class OfflineOCR(InfererModule, ModelWrapper):
        _MODEL_SUB_DIR = "ocr"

        def __init__(self):
            InfererModule.__init__(self)
            ModelWrapper.__init__(self)

        def _generate_text_direction(self, bboxes):
            yield from generate_text_direction(bboxes)

        async def recognize(self, image, textlines, config, verbose: bool = False):
            return await self.infer(image, textlines, config, verbose)

    class OfflineInpainter(InfererModule, ModelWrapper):
        _MODEL_SUB_DIR = "inpainting"

        def __init__(self):
            InfererModule.__init__(self)
            ModelWrapper.__init__(self)

        async def inpaint(self, image, mask, config, inpainting_size: int = 1024, verbose: bool = False):
            return await self.infer(image, mask, config, inpainting_size, verbose)

    @dataclass
    class OcrConfig:
        prob: Optional[float] = None
        ignore_bubble: int = 0
        min_text_length: int = 0

    @dataclass
    class InpainterConfig:
        inpainting_size: int = 2048
        inpainting_precision: str = "bf16"   # ignored: this path always computes at fp32 accuracy


def chunks(lst, n):
    for i in range(0, len(lst), n):
        yield lst[i:i + n]

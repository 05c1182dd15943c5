"""CPU: the `default` detector's plugin surface (no compute calls).  `register(default_detector=True)` against stand-ins for the
reference's registries (detection/__init__.py:12-27, config.py Detector enum), and the plugin's reference-facing attributes."""
import asyncio
import enum
import os
import sys
import types

import numpy as np
import pytest

from mit_b200 import compat, plugins


def _standin_registries(monkeypatch):
    class Detector(enum.Enum):
        default = "default"
        dbconvnext = "dbconvnext"

    class Ocr(enum.Enum):
        ocr48px_ctc = "48px_ctc"

    class Inpainter(enum.Enum):
        lama_mpe = "lama_mpe"
        lama_large = "lama_large"

    class Old:
        pass

    det = types.ModuleType("manga_translator.detection")
    det.DETECTORS, det.detector_cache = {Detector.default: Old, Detector.dbconvnext: Old}, {Detector.default: Old(), Detector.dbconvnext: Old()}
    ocr = types.ModuleType("manga_translator.ocr")
    ocr.OCRS, ocr.ocr_cache = {Ocr.ocr48px_ctc: Old}, {}
    inp = types.ModuleType("manga_translator.inpainting")
    inp.INPAINTERS, inp.inpainter_cache = {Inpainter.lama_mpe: Old, Inpainter.lama_large: Old}, {}
    cfg = types.ModuleType("manga_translator.config")
    cfg.Detector, cfg.Ocr, cfg.Inpainter = Detector, Ocr, Inpainter
    root = types.ModuleType("manga_translator")
    root.detection, root.ocr, root.inpainting, root.config = det, ocr, inp, cfg
    for name, mod in (("manga_translator", root), ("manga_translator.detection", det), ("manga_translator.ocr", ocr),
                      ("manga_translator.inpainting", inp), ("manga_translator.config", cfg)):
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.setattr(compat, "HAVE_REFERENCE", True)
    return Detector, det, Old


def test_register_default_detector_opt_in(monkeypatch):
    Detector, det, Old = _standin_registries(monkeypatch)
    plugins.register(default_detector=True)
    assert det.DETECTORS[Detector.default] is plugins.DefaultDetector
    assert det.DETECTORS[Detector.dbconvnext] is plugins.DBConvNextDetector
    assert Detector.default not in det.detector_cache and Detector.dbconvnext not in det.detector_cache
    obj = det.DETECTORS[Detector.default]()                    # the registry constructs it with no arguments
    with pytest.raises(Exception):
        asyncio.run(obj.infer(np.zeros((64, 64, 3), np.uint8), 512, 0.5, 0.7, 2.3))     # infer before load raises


def test_default_detector_plugin_surface(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    (tmp_path / "detect-20241225.ckpt").write_bytes(b"")
    before = sorted(os.listdir(tmp_path))
    det = plugins.DefaultDetector()
    assert sorted(os.listdir(tmp_path)) == before                # constructing it neither creates directories nor moves files
    m = plugins.DefaultDetector._MODEL_MAPPING["model"]
    assert m["url"].endswith("/beta-0.3/detect-20241225.ckpt") and m["file"] == "."
    assert m["hash"] == "67ce1c4ed4793860f038c71189ba9630a7756f7683b1ee5afb69ca0687dc502e"
    assert plugins.DefaultDetector._CKPT == "detect-20241225.ckpt"
    # injected weights are per class: setting the ConvNeXt detector's does not leak into the default detector
    plugins.DBConvNextDetector.set_state_dict({"x": None})
    try:
        assert plugins.DefaultDetector._injected is None
    finally:
        plugins.DBConvNextDetector.set_state_dict(None)
    import inspect
    assert inspect.signature(det._infer).parameters.keys() == inspect.signature(plugins.DBConvNextDetector._infer).parameters.keys() - {"self"}

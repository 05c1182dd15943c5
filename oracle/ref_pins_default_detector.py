"""TEST INFRASTRUCTURE -- recorded outputs of the reference's OWN default detector (detection/default.py, the network of
detection/default_utils/DBNet_resnet34.py) for tests/test_default_detector_pins.py.

Same conventions as oracle/ref_pins.py, whose helpers it reuses (digests, sampled positions, the duck-typed `_infer` call), written to
separate files so the existing pins stay untouched:

    tests/golden/reference_pins_default_detector.json   state-dict spec, output shapes, `_infer` quads / scores / mask digests
    tests/golden/reference_pins_default_detector.npz    the network's outputs at sampled positions

    python -m oracle.ref_pins_default_detector      # regenerate: needs the reference tree and torchvision, CPU only
    python -m oracle.ref_pins_default_detector --golden   # also (re)write the GPU tests' fixture tests/golden/dbnet_r34_256x512.npz
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

from . import dbnet_r34 as r34
from .ref_pins import ROOT, digest, sample_positions, state_dict_spec

GOLDEN_JSON = os.path.join(ROOT, "tests", "golden", "reference_pins_default_detector.json")
GOLDEN_NPZ = os.path.join(ROOT, "tests", "golden", "reference_pins_default_detector.npz")
FIXTURE = os.path.join(ROOT, "tests", "golden", "dbnet_r34_256x512.npz")
NET_CASES = ((256, 512, 1, 31), (512, 768, 1, 32))        # (h, w, n, seed) of oracle.cases.dbnet_case
GLUE_BIAS_SHIFT = -1.0                                     # added to conv_db.binarize.6.bias: random weights emit pixel noise otherwise

_cache = {}


def load():
    """(json dict, npz dict) of the recorded reference results."""
    if not _cache:
        _cache["j"] = json.load(open(GOLDEN_JSON))
        with np.load(GOLDEN_NPZ) as z:
            _cache["z"] = {k: z[k] for k in z.files}
    return _cache["j"], _cache["z"]


def glue_weights():
    sd = {k: v.clone() for k, v in r34.weights().items()}
    sd["conv_db.binarize.6.bias"] += GLUE_BIAS_SHIFT
    return sd


def fixture_case(n=1):
    """Input of the GPU fixture (regenerated from its seed, not stored): rectangular 256 x 512."""
    from oracle import cases
    return cases.dbnet_case(256, 512, n=n, seed=33)


def write_fixture():
    """tests/golden/dbnet_r34_256x512.npz from the oracle restatement (pinned above): db after the sigmoid, mask."""
    import torch
    torch.set_grad_enabled(False)
    _, x = fixture_case()
    db, mask = r34.forward(r34.weights(), x)
    np.savez_compressed(FIXTURE, db_sigmoid=db.sigmoid().numpy(), mask=mask.numpy())
    print(f"{FIXTURE}: {os.path.getsize(FIXTURE)} bytes")


def _reference(J, Z):
    import asyncio
    import importlib
    import logging
    import types
    import torch
    from oracle import cases, refload
    from oracle.ref_pins import _bind_third_party, _lines_json, detector_glue_pages
    torch.set_grad_enabled(False)
    refload.load()
    default = importlib.import_module("manga_translator.detection.default")
    J["state_dict_spec"] = state_dict_spec(default.TextDetectionDefault().state_dict())
    net = default.TextDetectionDefault().eval()
    net.load_state_dict(r34.weights(seed=2))
    for h, w, n, seed in NET_CASES:
        _, x = cases.dbnet_case(h, w, n=n, seed=seed)
        db, mask = net(x)
        for k, t in ((f"net_{h}x{w}_db", db), (f"net_{h}x{w}_mask", mask)):
            flat = t.numpy().reshape(-1)
            Z[k] = flat[sample_positions(flat.size)]
            J[k + "_shape"] = list(t.shape)
    _bind_third_party()
    sd = glue_weights()
    net = default.TextDetectionDefault().eval()
    net.load_state_dict(sd)
    default.MODEL = net
    me = types.SimpleNamespace(device="cpu", logger=logging.getLogger("ref-default-det"), model=net)
    J["detector_glue"] = []
    for page, detect_size in detector_glue_pages():
        r_lines, r_mask, _ = asyncio.run(default.DefaultDetector._infer(me, page, detect_size, 0.5, 0.6, 2.3))
        J["detector_glue"].append({"lines": _lines_json(r_lines), "mask_dtype": str(r_mask.dtype), "mask": digest(r_mask)})


def main():
    import warnings
    from oracle import refload
    warnings.filterwarnings("ignore")
    for p in (ROOT, os.path.join(ROOT, "manga-image-translator_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    if not refload.available():
        raise SystemExit(f"reference tree not found under {refload.REF_ROOT}")
    J, Z = {}, {}
    _reference(J, Z)
    json.dump(J, open(GOLDEN_JSON, "w"), separators=(",", ":"))
    np.savez_compressed(GOLDEN_NPZ, **Z)
    print(f"{GOLDEN_JSON}: {os.path.getsize(GOLDEN_JSON)} bytes, {GOLDEN_NPZ}: {os.path.getsize(GOLDEN_NPZ)} bytes")
    if "--golden" in sys.argv[1:]:
        write_fixture()


if __name__ == "__main__":
    main()

"""Pins the oracle restatement and the host glue on the unmodified reference modules: what the reference's own code returned on the
seeded inputs of oracle/ref_pins.py is recorded in tests/golden/reference_pins.{json,npz} (regenerate with `python -m oracle.ref_pins`
where the reference tree is available); here the oracle / product side is computed and compared with it."""
import numpy as np
import torch

from oracle import cases, nets, ref_pins, weights

torch.set_grad_enabled(False)


def test_state_dict_specs_match_reference():
    J, _ = ref_pins.load()
    spec = J["state_dict_specs"]
    assert spec["dbnet"] == ref_pins.state_dict_spec(weights.dbnet_weights())
    assert spec["ocr300"] == ref_pins.state_dict_spec(weights.ocr_weights(300))
    for nb in (9, 18):
        assert spec[f"lama{nb}"] == ref_pins.state_dict_spec(weights.lama_weights(nb))
    assert spec["mpe"] == ref_pins.state_dict_spec(weights.mpe_weights())
    assert spec["mpe_rel_pos_emb"] == ref_pins.digest(weights.mpe_weights()["rel_pos_emb.weight"].numpy())


def _sampled(t):
    flat = t.numpy().reshape(-1)
    return flat[ref_pins.sample_positions(flat.size)]


def test_dbnet_rectangular():
    J, Z = ref_pins.load()
    sd = weights.dbnet_weights(seed=2)
    _, x = cases.dbnet_case(256, 512, seed=21)
    o_db, o_mask = nets.dbnet_forward(sd, x)
    assert list(o_db.shape) == J["dbnet_rect_db_shape"] and list(o_mask.shape) == J["dbnet_rect_mask_shape"]
    assert np.abs(Z["dbnet_rect_db"] - _sampled(o_db)).max() < 1e-4 and np.abs(Z["dbnet_rect_mask"] - _sampled(o_mask)).max() < 1e-5


def test_ocr_widths_and_decode():
    J, Z = ref_pins.load()
    V = 300
    sd = weights.ocr_weights(V, seed=3)
    for wp in (143, 200, 331):
        rec = J["ocr_widths"][str(wp)]
        _, x = cases.ocr_case(3, wp, seed=wp)
        ol, oc = nets.ocr_forward(sd, x)
        assert list(ol.shape) == rec["logits_shape"]
        assert np.abs(Z[f"ocr_logits_{wp}"] - _sampled(ol)).max() < 1e-4 and np.abs(Z[f"ocr_colors_{wp}"] - oc.numpy()).max() < 1e-5
        idx, lp, col = nets.ocr_top1(sd, x)
        mine = nets.ctc_greedy(idx.numpy(), lp.numpy(), col.numpy())
        if rec["margin_ok"]:
            assert rec["decode"] == [[c[0] for c in l] for l in mine]


def test_lama_mpe_tables_random_masks():
    J, _ = ref_pins.load()
    masks = ref_pins.mpe_masks()
    assert len(masks) == len(J["mpe_tables"])
    for m, want in zip(masks, J["mpe_tables"]):
        orel, odirect = nets.mpe_tables(m)
        assert ref_pins.digest(orel) == want["rel"] and ref_pins.digest(odirect) == want["direct"]


def test_lama_odd_spectrum_sizes():
    _, Z = ref_pins.load()
    sd, msd = weights.lama_weights(9, seed=4), weights.mpe_weights(seed=4)
    img, mask = cases.lama_case(88, 120, seed=41)   # bottleneck 11x15: odd FFT lengths
    rel, direct = nets.mpe_tables(mask[0, 0].numpy())
    o = nets.lama_forward(sd, msd, img, mask, torch.from_numpy(rel)[None], torch.from_numpy(direct)[None])
    assert np.abs(Z["lama_odd"] - o.numpy()).max() < 2e-5


# ---------------------------------------------------------------------------------------------------------------------
# The three `_infer` glue paths: oracle/pipeline_ref.py (what the GPU plugin tests compare the product with) against the reference's own
# `_infer` methods, recorded from an unmodified run on the CPU with a duck-typed `self` and the absent third-party libraries bound to
# the repo's restatements (pyclipper -> Clipper 6.4.2 restatement, shapely -> geometry restatements).  Closes the loop: reference
# `_infer` == pipeline_ref here, plugin == pipeline_ref on the GPU.
def test_detector_infer_glue_equals_reference_code():
    from oracle import pipeline_ref
    J, _ = ref_pins.load()
    sd = ref_pins.detector_glue_weights()
    for (page, detect_size), want in zip(ref_pins.detector_glue_pages(), J["detector_glue"]):
        o_lines, o_mask, _, _ = pipeline_ref.detector_infer(sd, page, detect_size, 0.5, 0.6, 2.3)
        assert len(want["lines"]) == len(o_lines) and len(o_lines) > 3
        for a, b in zip(want["lines"], o_lines):
            assert np.array_equal(np.array(a["pts"]), b.pts) and a["prob"] == b.prob and a["direction"] == b.direction
        assert want["mask_dtype"] == "uint8" and ref_pins.digest(o_mask) == want["mask"]


def test_ocr_infer_glue_equals_reference_code():
    from mit_b200 import synth
    from mit_b200.host import geometry
    from oracle import pipeline_ref
    J, _ = ref_pins.load()
    V = cases.OCR_VOCAB_SMALL
    dictionary = weights.synthetic_dictionary(V)
    sd = weights.ocr_weights(V)
    page, boxes, _ = synth.make_page(3, 512, 384, 6)
    r_out = J["ocr_glue"]
    o_out = pipeline_ref.ocr_infer(sd, dictionary, page, [geometry.Quadrilateral(b.copy(), "", 1.0) for b in boxes], 0.0)
    assert len(r_out) == len(o_out) >= 4
    for a, b in zip(r_out, o_out):
        assert np.array_equal(np.array(a["pts"]), b.pts) and a["text"] == b.text and len(a["text"]) > 0
        assert abs(a["prob"] - b.prob) < 1e-4 * max(a["prob"], 1e-30)            # the two fp32 network evaluations differ by ~1e-5 in log-probability
        assert tuple(a["colors"]) == (b.fg_r, b.fg_g, b.fg_b, b.bg_r, b.bg_g, b.bg_b)


def test_inpainter_infer_glue_equals_reference_code():
    from oracle import pipeline_ref
    _, Z = ref_pins.load()
    sd, msd = weights.lama_weights(9), weights.mpe_weights()
    page, mask, sizes = ref_pins.inpainter_glue_case()
    for size in sizes:                                            # no resize; keep-aspect resize + back
        r = Z[f"inpainter_glue_{size}"]
        o, _ = pipeline_ref.lama_infer(sd, msd, page.copy(), mask.copy(), size)
        assert r.dtype == o.dtype == np.uint8 and r.shape == page.shape
        d = np.abs(r.astype(int) - o.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 1e-3, (int(d.max()), float((d > 0).mean()))     # x*255 truncation of fp32 values 2e-5 apart


def test_common_detector_detect_equals_reference_code():
    """D12: the stand-in `CommonDetector.detect` of mit_b200.compat (border for small pages, rotation, inversion, gamma correction,
    auto-rotation; used when the reference package cannot be imported) against the reference's own `detection/common.py` code, both
    wrapped around the same stub `_detect` (oracle/ref_pins.py): identical images handed to `_detect`, text lines, raw mask and mask
    for every combination of the switches."""
    import asyncio
    import importlib.util
    import sys
    from mit_b200 import compat as _compat_loaded
    from mit_b200.host import geometry
    J, _ = ref_pins.load()
    # a second copy of mit_b200/compat.py imported while `manga_translator` is hidden: that is the stand-in the GPU box gets
    hidden = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "manga_translator" or k.startswith("manga_translator.")}
    sys.modules["manga_translator"] = None                       # makes `import manga_translator...` raise ImportError
    try:
        spec = importlib.util.spec_from_file_location("mit_b200._compat_standin", _compat_loaded.__file__)
        compat = importlib.util.module_from_spec(spec)
        sys.modules["mit_b200._compat_standin"] = compat
        spec.loader.exec_module(compat)
    finally:
        del sys.modules["manga_translator"]
        sys.modules.update(hidden)
    assert not compat.HAVE_REFERENCE

    class OurDet(compat.OfflineDetector):
        _detect = ref_pins.detector_stub(geometry.Quadrilateral)

        async def _load(self, device):
            pass

        async def _unload(self):
            pass

        async def _infer(self, *a, **k):
            raise AssertionError("not used: `_detect` is stubbed")

    cases_ = ref_pins.common_detector_cases()
    assert len(cases_) == len(J["common_detector"])
    for (h, w, img, sw), want in zip(cases_, J["common_detector"]):
        o = OurDet()
        o.seen = []
        ot, oraw, omask = asyncio.run(o.detect(img.copy(), 1024, 0.5, 0.7, 2.3, *sw))
        assert want["seen"] == [ref_pins.digest(a) for a in o.seen], (h, w, sw)
        assert want["lines"] == (ref_pins.digest(np.stack([b.pts for b in ot])) if ot else None)
        assert want["raw"] == ref_pins.digest(oraw) and want["mask"] == ref_pins.digest(omask)

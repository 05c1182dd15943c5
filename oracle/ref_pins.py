"""TEST INFRASTRUCTURE -- recorded outputs of the reference's OWN code for the pinning tests.

The tests that pin the oracle restatement and the host ports on the reference (tests/test_oracle_vs_reference.py, the reference
tests of tests/test_host.py, tests/test_mask_refine.py and tests/test_textline_merge.py) compare against what the unmodified
reference modules returned on the seeded inputs built here, stored in tests/golden/reference_pins.json (structured results, and
truncated SHA-256 digests of arrays that are compared for equality) and tests/golden/reference_pins.npz (arrays compared with a tolerance;
page-sized ones as a fixed seeded sample of positions, see `sample_positions`).  The inputs are built by the functions below, which
the tests call too, so both sides see the same data.

    python -m oracle.ref_pins      # regenerate: needs the reference tree (oracle/refload.py), CPU only, about a minute

Regeneration binds the reference's absent third-party libraries (pyclipper, shapely, pydensecrf) to the repo's restatements exactly
as the tests always did; those restatements stay unpinned themselves.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import types

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_JSON = os.path.join(ROOT, "tests", "golden", "reference_pins.json")
GOLDEN_NPZ = os.path.join(ROOT, "tests", "golden", "reference_pins.npz")
SAMPLE = 20000                      # positions kept of a page-sized float output


def digest(a) -> str:
    """First 128 bits of the SHA-256 of an array's dtype, shape and bytes."""
    a = np.ascontiguousarray(np.asarray(a))
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()[:32]


def sample_positions(n: int, k: int = SAMPLE) -> np.ndarray:
    """Fixed positions into a flattened array of n elements (all of them when n <= k)."""
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.default_rng(n).choice(n, size=k, replace=False))


_cache = {}


def load():
    """(json dict, npz dict) of the recorded reference results."""
    if not _cache:
        _cache["j"] = json.load(open(GOLDEN_JSON))
        with np.load(GOLDEN_NPZ) as z:
            _cache["z"] = {k: z[k] for k in z.files}
    return _cache["j"], _cache["z"]


# ================================================================================================= inputs (shared with the tests)
def state_dict_spec(sd) -> str:
    """Digest of a state dict's parameter names and shapes (buffers the loaders do not fill excluded)."""
    spec = {k: list(v.shape) for k, v in sd.items() if "num_batches_tracked" not in k and not k.endswith("pe.pe")}
    return hashlib.sha256(json.dumps(spec, sort_keys=True).encode()).hexdigest()[:32]


def mpe_masks():
    rng = np.random.default_rng(5)
    out = []
    for (h, w) in ((256, 256), (200, 312), (64, 48)):
        m = np.zeros((h, w), np.float32)
        for _ in range(4):
            y, x = rng.integers(0, h - 8), rng.integers(0, w - 8)
            m[y:y + rng.integers(4, h // 2), x:x + rng.integers(4, w // 2)] = 1
        out.append(m)
    return out + [np.zeros((64, 64), np.float32), np.ones((64, 64), np.float32)]   # all-hole / no-hole masks terminate


def detector_glue_pages():
    from mit_b200 import synth
    return ((synth.make_page(5, 512, 384, 6)[0], 512), (synth.make_page(4, 384, 384, 5)[0], 512))      # pad path; upscale path


def detector_glue_weights():
    from oracle import weights
    sd = {k: v.clone() for k, v in weights.dbnet_weights().items()}
    sd["conv_db.binarize.4.bias"] -= 1.0
    return sd


def inpainter_glue_case():
    rng = np.random.default_rng(6)
    page = rng.integers(0, 256, (200, 152, 3), dtype=np.uint8)
    mask = np.zeros((200, 152), np.uint8)
    mask[20:50, 10:120] = 255
    mask[120:180, 60:90] = 255
    mask[100:104, 5:40] = 130
    mask[10, 10] = 127                                            # the 127 / 128 threshold quirk (SURVEY I2)
    return page, mask, (1024, 128)                                # no resize; keep-aspect resize + back


def detector_stub(quad_cls):
    """`_detect` stand-in for CommonDetector.detect: records the images it is given, returns seeded lines / masks."""
    async def _detect(self, image, detect_size, text_threshold, box_threshold, unclip_ratio, verbose=False):
        self.seen.append(image.copy())
        h, w = image.shape[:2]
        rng = np.random.default_rng(h * 7919 + w)
        lines = []
        for _ in range(6):
            x0, y0 = int(rng.integers(0, w - 40)), int(rng.integers(0, h - 40))
            bw, bh = int(rng.integers(12, 120)), int(rng.integers(8, 60))
            lines.append(quad_cls(np.array([[x0, y0], [x0 + bw, y0], [x0 + bw, y0 + bh], [x0, y0 + bh]]), "", 0.9))
        lines.append(quad_cls(np.array([[5, 5], [6, 5], [6, 6], [5, 6]]), "", 0.5))          # area 1: filtered
        raw = (rng.random((h, w)) * 255).astype(np.uint8)
        return lines, raw, (rng.random((h, w)) > 0.5).astype(np.uint8) * 255
    return _detect


def common_detector_cases():
    """(h, w, image, switches) for every page size and every combination of invert / gamma / rotate / auto-rotate."""
    import itertools
    rng = np.random.default_rng(2)
    out = []
    for (h, w) in ((300, 200), (520, 450), (380, 700)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for sw in itertools.product((False, True), repeat=4):
            out.append((h, w, img, sw))
    return out


def quadrilateral_cases():
    from mit_b200 import synth
    rng = np.random.default_rng(4)
    page, boxes, _ = synth.make_page(1, 1024, 768, 10)
    bs = [b[rng.permutation(4)] for b in boxes + [np.array([[100, 100], [400, 130], [390, 190], [95, 160]]),
                                                   np.array([[50, 50], [90, 60], [70, 400], [30, 390]])]]
    return page, bs


def rearrange_fwd(batch, device=None):
    batch = np.asarray(batch).astype(np.float32)
    s = batch.shape[1]
    db = np.stack([batch[..., 0] / 255.0, batch[..., 1] / 255.0], 1).astype(np.float32)
    mask = np.stack([cv2.resize(b[..., 2], (s // 2, s // 2)) / 255.0 for b in batch])[:, None].astype(np.float32)
    return db, mask


def rearrange_images():
    rng = np.random.default_rng(0)
    return [cv2.GaussianBlur(rng.integers(0, 256, shape, dtype=np.uint8), (0, 0), 5) for shape in ((3000, 500, 3), (500, 3300, 3), (1024, 768, 3))]


def detector_helper_inputs():
    rng = np.random.default_rng(5)
    prob = cv2.GaussianBlur(rng.random((120, 160)).astype(np.float32), (0, 0), 4)
    cnts, _ = cv2.findContours(((prob > prob.mean()) * 255).astype(np.uint8), cv2.RETR_LIST, cv2.CHAIN_APPROX_SIMPLE)
    contours = [c.squeeze(1) for c in cnts[:10] if len(c.squeeze(1)) >= 3]
    img = rng.integers(0, 256, (300, 200, 3), dtype=np.uint8)
    return prob, contours, img, (512, 256, 300)


def boxes_from_prob_input():
    rng = np.random.default_rng(11)
    prob = (0.05 * rng.random((400, 600))).astype(np.float32)
    for k in range(14):                                        # rotated / thin / tiny blobs, some below box_thresh
        cx, cy, w, h, ang = rng.integers(40, 560), rng.integers(40, 360), rng.integers(3, 120), rng.integers(3, 40), rng.uniform(0, 180)
        pts = cv2.boxPoints(((float(cx), float(cy)), (float(w), float(h)), float(ang))).astype(np.int32)
        cv2.fillPoly(prob, [pts], float(rng.uniform(0.55, 0.99)))
    return prob, ((600, 400), (1500, 1000))


def mask_refine_page(seed=3, h=768, w=576, n=8):
    from mit_b200 import synth
    page, boxes, _ = synth.make_page(seed, h, w, n)
    raw = cv2.dilate(((page[..., 0] < 100) * 255).astype(np.uint8), np.ones((3, 3), np.uint8))
    return page, boxes, raw


def mask_refine_regions(boxes, k=2):
    return [types.SimpleNamespace(lines=[b.astype(np.float64) for b in boxes[i:i + k]]) for i in range(0, len(boxes), k)]


def scaled_line_boxes():
    _, boxes, _ = mask_refine_page()
    return [b * (2.0 / 3.0) for b in boxes + [np.array([[10, 20], [200, 35], [195, 80], [5, 66]])]]


def mask_dispatch_cases():
    """(page, regions, raw, dilation_offset) of the dispatch pin: two pages plus a line without components."""
    out = []
    for seed, (h, w, n), offset in ((3, (768, 576, 8), 0), (9, (640, 480, 6), 20)):
        page, boxes, raw = mask_refine_page(seed, h, w, n)
        regions = mask_refine_regions(boxes) + [types.SimpleNamespace(lines=[np.array([[5.0, 5.0], [60.0, 5.0], [60.0, 30.0], [5.0, 30.0]])])]
        out.append((page, regions, raw, offset))
    return out


MERGE_PARAMS = (dict(aspect_ratio_tol=1), dict(aspect_ratio_tol=1.3, font_size_ratio_tol=2, char_gap_tolerance=1, char_gap_tolerance2=3))


def merge_predicate_sets():
    """Point lists of every known-answer case of tests/golden/textline_merge.json plus a set of rotated random quads."""
    cases = json.load(open(os.path.join(ROOT, "tests", "golden", "textline_merge.json")))["cases"]
    rng = np.random.default_rng(8)
    sets = [[np.array(l) for l in c["lines"]] for c in cases]
    rnd = []
    for t in range(60):
        cx, cy = rng.uniform(200, 500), rng.uniform(200, 500)
        ww, hh = rng.uniform(30, 200), rng.uniform(12, 40)
        if t % 3 == 0:
            ww, hh = hh, ww
        ang = rng.uniform(-0.5, 0.5) if t % 2 else 0.0
        c, s = np.cos(ang), np.sin(ang)
        rnd.append((np.array([[-ww / 2, -hh / 2], [ww / 2, -hh / 2], [ww / 2, hh / 2], [-ww / 2, hh / 2]]) @ np.array([[c, s], [-s, c]]) + [cx, cy]).astype(np.int64))
    sets.append(rnd)
    return sets


def merge_pages():
    """12 random clustered pages of rotated lines: [(point list, colours)]."""
    rng = np.random.default_rng(21)
    pages = []
    for page in range(12):
        pts_list = []
        for blk in range(int(rng.integers(2, 5))):           # a few "speech bubbles" of stacked lines + stray lines
            bx, by = rng.uniform(100, 900), rng.uniform(100, 700)
            vertical = rng.random() < 0.5
            fs = rng.uniform(18, 40)
            ang = rng.uniform(-0.12, 0.12) if rng.random() < 0.4 else 0.0
            for k in range(int(rng.integers(1, 6))):
                ln = rng.uniform(60, 260)
                w, h = (fs, ln) if vertical else (ln, fs)
                cx, cy = (bx - k * fs * rng.uniform(1.05, 1.6), by + rng.uniform(-8, 8)) if vertical else (bx + rng.uniform(-8, 8), by + k * fs * rng.uniform(1.05, 1.6))
                c, s = np.cos(ang), np.sin(ang)
                pts_list.append((np.array([[-w / 2, -h / 2], [w / 2, -h / 2], [w / 2, h / 2], [-w / 2, h / 2]]) @ np.array([[c, s], [-s, c]]) + [cx, cy]).astype(np.int64))
        cols = [tuple(int(v) for v in rng.integers(0, 256, 6)) for _ in pts_list]
        pages.append((pts_list, cols))
    return pages


# ================================================================================================= the reference side (regeneration)
def _shapely_standins():
    from mit_b200.host import geometry

    class Polygon:
        def __init__(self, pts):
            self.p = np.asarray(pts, dtype=np.float64).reshape(-1, 2)
            self.area, self.length = geometry.polygon_area(self.p), geometry.polygon_perimeter(self.p)

        @property
        def convex_hull(self):
            return Polygon(geometry._hull(self.p))

        def distance(self, other):
            return geometry.polygon_distance(self.p, other.p)
    return Polygon


def _bind_third_party():
    """pyclipper -> the Clipper 6.4.2 restatement, shapely Polygon / MultiPoint -> the geometry restatements."""
    import importlib
    from mit_b200.host import det_post
    G = importlib.import_module("manga_translator.utils.generic")
    du = importlib.import_module("manga_translator.detection.default_utils.dbnet_utils")

    class _Offset:
        def AddPath(self, box, jt, et):
            self.box = box

        def Execute(self, d):
            return [det_post.clipper_offset_round(self.box, d)]
    Polygon = _shapely_standins()
    du.pyclipper = type("pc", (), dict(PyclipperOffset=_Offset, JT_ROUND=1, ET_CLOSEDPOLYGON=2))
    du.Polygon = G.Polygon = G.MultiPoint = Polygon


def _lines_json(lines):
    return [{"pts": np.asarray(q.pts).tolist(), "prob": float(q.prob), "direction": q.direction} for q in lines]


def _oracle_vs_reference(R, J, Z):
    import asyncio
    import logging
    import torch
    from oracle import cases, weights
    torch.set_grad_enabled(False)
    # state-dict layouts
    spec = {"dbnet": state_dict_spec(R["det"].DBNetConvNext().state_dict()), "ocr300": state_dict_spec(R["ocr"].OCR(["x"] * 300, 768).state_dict())}
    for nb in (9, 18):
        lf = R["lama"].LamaFourier(build_discriminator=False, use_mpe=nb == 9, large_arch=nb == 18)
        spec[f"lama{nb}"] = state_dict_spec(lf.generator.state_dict())
        if nb == 9:
            spec["mpe"] = state_dict_spec(lf.mpe.state_dict())
            spec["mpe_rel_pos_emb"] = digest(lf.mpe.rel_pos_emb.weight.numpy())
    J["state_dict_specs"] = spec
    # DBNet on a rectangular input
    sd = weights.dbnet_weights(seed=2)
    net = R["det"].DBNetConvNext().eval()
    net.load_state_dict(sd)
    _, x = cases.dbnet_case(256, 512, seed=21)
    r_db, r_mask = net(x)
    for k, t in (("dbnet_rect_db", r_db), ("dbnet_rect_mask", r_mask)):
        flat = t.numpy().reshape(-1)
        Z[k] = flat[sample_positions(flat.size)]
        J[k + "_shape"] = list(t.shape)
    # OCR widths and decode
    V = 300
    sd = weights.ocr_weights(V, seed=3)
    ocr = R["ocr"].OCR(weights.synthetic_dictionary(V), 768).eval()
    ocr.load_state_dict(sd, strict=False)
    J["ocr_widths"] = {}
    for wp in (143, 200, 331):
        _, x = cases.ocr_case(3, wp, seed=wp)
        rl, rc = ocr(x)
        flat = rl.numpy().reshape(-1)
        Z[f"ocr_logits_{wp}"] = flat[sample_positions(flat.size)]
        Z[f"ocr_colors_{wp}"] = rc.numpy()
        top2 = rl.topk(2, dim=-1).values
        J["ocr_widths"][str(wp)] = {"logits_shape": list(rl.shape), "margin_ok": bool((top2[..., 0] - top2[..., 1]).min() > 1e-3),
                                    "decode": [[int(c[0]) for c in l] for l in ocr.decode(x, [0] * 3, 0)]}
    # MPE tables
    lf = R["lama"].LamaFourier(build_discriminator=False, use_mpe=True)
    J["mpe_tables"] = []
    for m in mpe_masks():
        rel, _, direct = lf.load_masked_position_encoding(m)
        J["mpe_tables"].append({"rel": digest(rel), "direct": digest(direct)})
    # LaMa at odd FFT lengths
    sd, msd = weights.lama_weights(9, seed=4), weights.mpe_weights(seed=4)
    lf = R["lama"].LamaFourier(build_discriminator=False, use_mpe=True)
    lf.generator.load_state_dict(sd)
    lf.mpe.load_state_dict(msd)
    lf.eval()
    img, mask = cases.lama_case(88, 120, seed=41)
    Z["lama_odd"] = lf(img.clone(), mask).numpy()
    # the three `_infer` glue paths, run unmodified with a duck-typed `self`
    _bind_third_party()
    det = R["det"]
    sd = detector_glue_weights()
    net = det.DBNetConvNext().eval()
    net.load_state_dict(sd)
    det.MODEL = net
    me = types.SimpleNamespace(device="cpu", logger=logging.getLogger("ref-det"), model=net)
    J["detector_glue"] = []
    for page, detect_size in detector_glue_pages():
        r_lines, r_mask, _ = asyncio.run(det.DBConvNextDetector._infer(me, page, detect_size, 0.5, 0.6, 2.3))
        J["detector_glue"].append({"lines": _lines_json(r_lines), "mask_dtype": str(r_mask.dtype), "mask": digest(r_mask)})
    from mit_b200 import synth
    Vs = cases.OCR_VOCAB_SMALL
    model = R["ocr"].OCR(weights.synthetic_dictionary(Vs), 768).eval()
    model.load_state_dict(weights.ocr_weights(Vs), strict=False)
    common = sys.modules["manga_translator.ocr.common"]
    page, boxes, _ = synth.make_page(3, 512, 384, 6)
    me = types.SimpleNamespace(device="cpu", use_gpu=False, logger=logging.getLogger("ref-ocr"), model=model)
    me._generate_text_direction = lambda bboxes: common.CommonOCR._generate_text_direction(me, bboxes)
    r_out = asyncio.run(R["ocr"].Model48pxCTCOCR._infer(me, page, [R["utils"].Quadrilateral(b.copy(), "", 1.0) for b in boxes],
                                                        types.SimpleNamespace(ignore_bubble=0, prob=0.0), False))
    J["ocr_glue"] = [{"pts": np.asarray(a.pts).tolist(), "text": a.text, "prob": float(a.prob),
                      "colors": [int(v) for v in (a.fg_r, a.fg_g, a.fg_b, a.bg_r, a.bg_g, a.bg_b)]} for a in r_out]
    lama = R["lama"]
    lf = lama.LamaFourier(build_discriminator=False, use_mpe=True)
    lf.generator.load_state_dict(weights.lama_weights(9))
    lf.mpe.load_state_dict(weights.mpe_weights())
    lf.eval()
    me = types.SimpleNamespace(device="cpu", logger=logging.getLogger("ref-inp"), model=lf)
    page, mask, sizes = inpainter_glue_case()
    for size in sizes:
        Z[f"inpainter_glue_{size}"] = asyncio.run(lama.LamaMPEInpainter._infer(me, page.copy(), mask.copy(),
                                                                               types.SimpleNamespace(inpainting_precision="fp32"), size, False))
    # CommonDetector.detect around the stub `_detect`
    import importlib
    rc = importlib.import_module("manga_translator.detection.common")

    class RefDet(rc.CommonDetector):
        _detect = detector_stub(R["utils"].Quadrilateral)
    J["common_detector"] = []
    for h, w, img, sw in common_detector_cases():
        r = RefDet()
        r.seen = []
        rt, rraw, rmask = asyncio.run(r.detect(img.copy(), 1024, 0.5, 0.7, 2.3, *sw))
        J["common_detector"].append({"seen": [digest(s) for s in r.seen], "lines": digest(np.stack([np.asarray(q.pts) for q in rt])) if rt else None,
                                     "raw": digest(rraw), "mask": digest(rmask)})


def _host(R, J, Z):
    import importlib
    U = R["utils"]
    page, bs = quadrilateral_cases()
    J["quadrilateral"] = []
    for b in bs:
        q = U.Quadrilateral(b, "", 1.0)
        J["quadrilateral"].append({"pts": np.asarray(q.pts).tolist(), "direction": q.direction, "aspect_ratio": float(q.aspect_ratio),
                                   "font_size": float(q.font_size), "aabb": [int(v) for v in (q.aabb.x, q.aabb.y, q.aabb.w, q.aabb.h)],
                                   "axis_aligned": bool(q.is_approximate_axis_aligned), "angle": float(q.angle),
                                   "regions": {d: digest(q.get_transformed_region(page, d, 48)) for d in ("h", "v")}})
    J["rearrange"] = []
    for img in rearrange_images():
        r = U.det_rearrange_forward(img, rearrange_fwd, 1024, 4)
        J["rearrange"].append(None if r[0] is None else [digest(r[0]), digest(r[1])])
    du = importlib.import_module("manga_translator.detection.default_utils.dbnet_utils")
    ip = importlib.import_module("manga_translator.detection.default_utils.imgproc")
    rep = du.SegDetectorRepresenter(0.5, 0.7, unclip_ratio=2.3)
    prob, contours, img, sizes = detector_helper_inputs()
    J["detector_helpers"] = {"mini_boxes": [], "scores": [], "resize": []}
    for c in contours:
        box, sside = rep.get_mini_boxes(c)
        J["detector_helpers"]["mini_boxes"].append({"box": np.array(box, np.float64).tolist(), "sside": float(sside)})
        J["detector_helpers"]["scores"].append(float(rep.box_score_fast(prob, c)))
    for size in sizes:
        b = ip.resize_aspect_ratio(img, size, cv2.INTER_LINEAR, mag_ratio=1)
        J["detector_helpers"]["resize"].append({"img": digest(b[0]), "rest": [float(v) if np.ndim(v) == 0 else list(v) for v in b[1:]]})
    _bind_third_party()
    rep = du.SegDetectorRepresenter(0.5, 0.7, unclip_ratio=2.3)
    prob, sizes = boxes_from_prob_input()
    for (dw, dh) in sizes:
        rb, rs = rep.boxes_from_bitmap(prob, prob > 0.5, dw, dh)
        Z[f"boxes_from_prob_{dw}_boxes"], Z[f"boxes_from_prob_{dw}_scores"] = np.asarray(rb), np.asarray(rs)


def _load_reference_mask_refinement():
    """The reference's OWN mask_refinement package (`__init__.py` + `text_mask_utils.py`, unmodified) with its two absent third-party
    dependencies bound to the oracle's restatements: shapely.geometry.Polygon (area / intersection / distance / centroid) and
    pydensecrf (DenseCRF2D, unary_from_softmax)."""
    import importlib.util
    from oracle import mask_refine_ref as MR
    from oracle import refload
    refload.load()

    class _Pt:
        def __init__(self, x, y):
            self.x, self.y = x, y

    class Polygon:
        def __init__(self, pts):
            self.p = np.asarray(pts, dtype=np.float64).reshape(-1, 2)

        @property
        def area(self):
            return MR.poly_area(self.p) if len(self.p) >= 3 else 0.0

        @property
        def centroid(self):                                     # only ever asked of the component rectangle
            return _Pt(float(self.p[:, 0].mean()), float(self.p[:, 1].mean()))

        def intersection(self, other):                          # `other` is the axis-aligned component rectangle
            x0, y0, x1, y1 = other.p[:, 0].min(), other.p[:, 1].min(), other.p[:, 0].max(), other.p[:, 1].max()
            return Polygon(np.asarray(MR.clip_poly_rect(self.p, x0, y0, x1, y1)).reshape(-1, 2))

        def distance(self, pt):
            return MR.point_poly_distance(self.p, pt.x, pt.y)

    class DenseCRF2D:
        def __init__(self, w, h, n):
            self.w, self.h, self.n = w, h, n

        def setUnaryEnergy(self, u):
            self.u = np.asarray(u, dtype=np.float32)

        def addPairwiseGaussian(self, sxy, compat, kernel=None, normalization=None):
            self.g = (float(sxy), float(compat))

        def addPairwiseBilateral(self, sxy, srgb, rgbim, compat, kernel=None, normalization=None):
            self.b, self.rgb = (float(sxy), float(srgb), float(compat)), np.asarray(rgbim)

        def inference(self, n):
            assert self.rgb.shape[:2] == (self.h, self.w)
            return MR.dense_crf_2d(self.rgb, self.u, n, self.g[0], self.g[1], self.b[0], self.b[1], self.b[2])

    geom = sys.modules["shapely.geometry"]
    geom.Polygon = Polygon
    dcrf = types.ModuleType("pydensecrf.densecrf")
    dcrf.DenseCRF2D, dcrf.DIAG_KERNEL, dcrf.NO_NORMALIZATION = DenseCRF2D, 1, 0
    putils = types.ModuleType("pydensecrf.utils")
    putils.unary_from_softmax = lambda sm, scale=None, clip=1e-5: (-np.log(np.clip(sm, clip, 1.0))).reshape([sm.shape[0], -1]).astype(np.float32)
    putils.compute_unary = None
    pkg = types.ModuleType("pydensecrf")
    pkg.__path__ = []
    pkg.densecrf, pkg.utils = dcrf, putils
    sys.modules.update({"pydensecrf": pkg, "pydensecrf.densecrf": dcrf, "pydensecrf.utils": putils})
    path = os.path.join(refload.REF_ROOT, "manga_translator", "mask_refinement")
    spec = importlib.util.spec_from_file_location("manga_translator.mask_refinement", os.path.join(path, "__init__.py"), submodule_search_locations=[path])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["manga_translator.mask_refinement"] = mod
    spec.loader.exec_module(mod)
    return mod


def _mask_refine(R, J, Z):
    import asyncio
    from oracle import mask_refine_ref as MR
    U = R["utils"]
    J["scaled_lines"] = []
    for b in scaled_line_boxes():
        r = MR._Line(U.Quadrilateral, b)
        J["scaled_lines"].append({"pts": np.asarray(r.pts).tolist(), "font_size": float(r.font_size), "aabb_xywh": np.asarray(r.aabb_xywh).tolist()})
    ref = _load_reference_mask_refinement()
    J["mask_dispatch"] = []
    for page, regions, raw, offset in mask_dispatch_cases():
        want = asyncio.run(ref.dispatch(regions, page, raw.copy(), "fit_text", offset, 0, False, 3))
        J["mask_dispatch"].append({"dtype": str(want.dtype), "mask": digest(want), "coverage": float((want > 0).mean())})


def _textline_merge(R, J, Z):
    import importlib.util
    import itertools
    from mit_b200.host import geometry
    from oracle import refload
    U = R["utils"]
    G = __import__("manga_translator.utils.generic", fromlist=["x"])
    common = sys.modules["manga_translator.ocr.common"]
    Polygon = _shapely_standins()
    G.Polygon = G.MultiPoint = Polygon
    # the merge predicate over every pair of every set, under both parameter sets (bit string per set and parameter set)
    J["merge_predicate"] = []
    for pts_list in merge_predicate_sets():
        ref = [U.Quadrilateral(p, "", 1.0) for p in pts_list]
        for r, p in zip(ref, pts_list):                        # the angled branch asks Quadrilateral.poly_distance (hull polygons)
            r.__dict__["polygon"] = Polygon(geometry._hull(geometry.Quadrilateral(p, "", 1.0).pts))
        J["merge_predicate"].append(["".join("1" if G.quadrilateral_can_merge_region(ref[u], ref[v], **params) else "0"
                                             for u, v in itertools.combinations(range(len(ref)), 2)) for params in MERGE_PARAMS])
    # merge_bboxes_text_region and the OCR direction graph on random pages
    path = os.path.join(refload.REF_ROOT, "manga_translator", "textline_merge", "__init__.py")
    spec = importlib.util.spec_from_file_location("manga_translator.textline_merge", path, submodule_search_locations=[os.path.dirname(path)])
    ref_merge = importlib.util.module_from_spec(spec)
    sys.modules["manga_translator.textline_merge"] = ref_merge
    spec.loader.exec_module(ref_merge)
    ref_merge.Polygon = Polygon
    J["merge_pages"] = []
    for pts_list, cols in merge_pages():
        ref = [U.Quadrilateral(p, f"t{i}", 0.9, *c) for i, (p, c) in enumerate(zip(pts_list, cols))]
        for q in ref:
            q.assigned_direction = q.direction
        regions = [[[ref.index(q) for q in tl], list(fg), list(bg)] for tl, fg, bg in ref_merge.merge_bboxes_text_region(ref, 1000, 800)]
        directions = [[ref.index(q), d] for q, d in common.CommonOCR._generate_text_direction(None, ref)]
        J["merge_pages"].append({"regions": regions, "directions": directions})


def main():
    import warnings
    from oracle import refload
    warnings.filterwarnings("ignore")
    for p in (ROOT, os.path.join(ROOT, "manga-image-translator_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    if not refload.available():
        raise SystemExit(f"reference tree not found under {refload.REF_ROOT}")
    R = refload.load()
    J, Z = {}, {}
    _oracle_vs_reference(R, J, Z)
    _host(R, J, Z)
    _mask_refine(R, J, Z)
    _textline_merge(R, J, Z)
    json.dump(J, open(GOLDEN_JSON, "w"), separators=(",", ":"))
    np.savez_compressed(GOLDEN_NPZ, **Z)
    print(f"{GOLDEN_JSON}: {os.path.getsize(GOLDEN_JSON)} bytes, {GOLDEN_NPZ}: {os.path.getsize(GOLDEN_NPZ)} bytes")


if __name__ == "__main__":
    main()

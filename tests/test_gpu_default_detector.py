"""The default detector (DBNet-ResNet34, detection/default.py) on the GPU: the network through the C ABI against the committed fixture
and the CPU oracle (pinned on the reference in tests/test_default_detector_pins.py), its new kernels against torch, and the
DefaultDetector plugin against the CPU restatement of the reference's `_infer`.  Bars: fp32 tensors within 1e-3, IoU >= 0.999 at
0.5 on db[:, 0] and the mask; max pool bit-exact."""
import asyncio
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from mit_b200 import MitbError, plugins, synth
from oracle import cases, weights
from oracle import dbnet_r34 as r34
from oracle import ref_pins_default_detector as pins

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
TOL = 1e-3


@pytest.fixture(scope="module")
def eng():
    from mit_b200.engine import get_engine
    e = get_engine("cuda:0")
    e.load_dbnet_r34(r34.weights())
    return e


def _err(a, b):
    return (torch.as_tensor(a).detach().cpu().float() - torch.as_tensor(b).float()).abs().max().item()


def _iou(a, b, thr=0.5):
    a, b = np.asarray(a) > thr, np.asarray(b) > thr
    u = (a | b).sum()
    return 1.0 if u == 0 else float((a & b).sum()) / float(u)


def _check(db, mask, r_db, r_mask, label):
    r_db, r_mask = torch.as_tensor(r_db), torch.as_tensor(r_mask)
    e_db, e_mask = _err(db, r_db), _err(mask, r_mask)
    i_db, i_mask = _iou(db[:, 0].cpu().numpy(), r_db[:, 0].numpy()), _iou(mask.cpu().numpy(), r_mask.numpy())
    print(f"dbnet_r34 {label}: db err {e_db:.2e} mask err {e_mask:.2e} IoU db {i_db:.5f} mask {i_mask:.5f}")
    assert e_db < TOL and e_mask < TOL and i_db >= 0.999 and i_mask >= 0.999


def _oracle(sd, x):
    db, mask = r34.forward(sd, x)
    return db.sigmoid(), mask


def test_network_fixture_oracle_and_u8(eng, golden_dir):
    g = np.load(os.path.join(golden_dir, "dbnet_r34_256x512.npz"))
    img, x = pins.fixture_case(n=2)                                  # image 0 is the fixture's input
    db, mask = eng.dbnet_r34_forward(x)
    _check(db[:1], mask[:1], g["db_sigmoid"], g["mask"], "fixture 256x512")
    _check(db, mask, *_oracle(r34.weights(), x), "oracle 2x256x512")
    db8, mask8 = eng.dbnet_r34_forward(torch.from_numpy(img))           # fused u8 normalisation = the fp32 entry
    assert _err(db8, db.cpu()) < 1e-6 and _err(mask8, mask.cpu()) < 1e-6
    _, x = cases.dbnet_case(512, 768, seed=34)                         # 2 x 3 map at 1/256
    db, mask = eng.dbnet_r34_forward(x)
    _check(db, mask, *_oracle(r34.weights(), x), "oracle 512x768")


def test_errors(eng):
    with pytest.raises(MitbError):
        eng.dbnet_r34_forward(torch.zeros(1, 3, 256, 384))           # w not a multiple of 256
    with pytest.raises(MitbError):
        eng.dbnet_r34_forward(torch.zeros(1, 3, 128, 256))           # h not a multiple of 256
    eng.unload_dbnet_r34()
    try:
        with pytest.raises(MitbError):
            eng.dbnet_r34_forward(torch.zeros(1, 3, 256, 256))       # forward before load
    finally:
        eng.load_dbnet_r34(r34.weights())


def test_exact_simt_path(eng, golden_dir):
    g = np.load(os.path.join(golden_dir, "dbnet_r34_256x512.npz"))
    _, x = pins.fixture_case()
    eng.set_tensor_cores(False)
    try:
        db, mask = eng.dbnet_r34_forward(x)
    finally:
        eng.set_tensor_cores(True)
    _check(db, mask, g["db_sigmoid"], g["mask"], "SIMT fixture")


def test_both_detectors_resident(eng, golden_dir):
    eng.load_dbnet(weights.dbnet_weights())
    try:
        g = np.load(os.path.join(golden_dir, "dbnet_256.npz"))
        _, x = cases.dbnet_case()
        db, mask = eng.dbnet_forward(x)
        _check(db, mask, g["db_sigmoid"], g["mask"], "ConvNeXt next to r34")
        g = np.load(os.path.join(golden_dir, "dbnet_r34_256x512.npz"))
        _, x = pins.fixture_case()
        db, mask = eng.dbnet_r34_forward(x)
        _check(db, mask, g["db_sigmoid"], g["mask"], "r34 next to ConvNeXt")
    finally:
        eng.unload_dbnet()


@pytest.mark.parametrize("shape", [(2, 64, 33, 47), (1, 3, 9, 8), (1, 64, 1, 1), (3, 20, 64, 64)])
def test_maxpool3x3s2_bit_exact(eng, shape):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(shape, generator=g) - 2.0                          # mostly negative: -inf padding matters
    y = eng.maxpool3x3s2(x).cpu()
    ref = F.max_pool2d(x, 3, 2, 1)
    assert y.shape == ref.shape and torch.equal(y, ref)


def test_stride2_stem_on_tensor_cores(eng):
    g = torch.Generator().manual_seed(7)
    for (n, h, w) in ((1, 97, 130), (2, 256, 192)):
        x = torch.randn(n, 3, h, w, generator=g)
        wt = torch.randn(64, 3, 7, 7, generator=g) * (1.0 / 147) ** 0.5
        b = torch.randn(64, generator=g) * 0.1
        y = eng.conv2d(x, wt, b, (2, 2), (3, 3))
        ref = F.conv2d(x, wt, b, stride=2, padding=3)
        assert y.shape == ref.shape and _err(y, ref) < TOL, _err(y, ref)

    def launches(stride, k, pad):
        x = torch.randn(1, 3, 128, 128, generator=g)
        before = eng.launches
        eng.conv2d(x, torch.randn(64, 3, k, k, generator=g) * 0.1, None, (stride, stride), (pad, pad))
        return eng.launches - before
    # the stem path is a split launch + the conv launch; the gather kernel (the ConvNeXt 4x4 s4 stem) is one launch
    s2, s1, s4 = launches(2, 7, 3), launches(1, 7, 3), launches(4, 4, 0)
    assert s2 == s1 == s4 + 1, (s2, s1, s4)


def test_full_size_2048x1536(eng):
    torch.set_num_threads(max(1, min(64, os.cpu_count() or 1)))
    sd = r34.weights()
    _, x = cases.dbnet_case(2048, 1536, seed=35)
    db, mask = eng.dbnet_r34_forward(x)
    _check(db, mask, *_oracle(sd, x), "2048x1536")


def _assert_same_detections(lines, r_lines, raw_mask, r_mask):
    """The bars of test_gpu_plugins._assert_same_detections: >= 95 % of the boxes identical, >= 97 % within 1 px, raw-mask IoU >= 0.999."""
    assert abs(len(lines) - len(r_lines)) <= max(1, len(r_lines) // 20), (len(lines), len(r_lines))
    ref_pts = [b.pts for b in r_lines]
    exact = sum(1 for a in lines if any(np.array_equal(a.pts, p) for p in ref_pts))
    near = sum(1 for a in lines if any(np.abs(a.pts - p).max() <= 1 for p in ref_pts))
    print(f"default detector boxes: {len(lines)} vs {len(r_lines)} reference, identical {exact}, within 1 px {near}")
    assert exact >= 0.95 * len(r_lines) and near >= 0.97 * len(r_lines), (exact, near, len(r_lines))
    inter = ((raw_mask > 127) & (r_mask > 127)).sum()
    union = ((raw_mask > 127) | (r_mask > 127)).sum()
    assert union == 0 or inter / union >= 0.999
    assert (np.abs(raw_mask.astype(int) - r_mask.astype(int)) > 1).mean() < 1e-3


def test_default_detector_plugin_matches_cpu_reference_path():
    sd = pins.glue_weights()
    plugins.DefaultDetector.set_state_dict(sd)
    det = plugins.DefaultDetector()
    try:
        with pytest.raises(Exception):
            asyncio.run(det.infer(np.zeros((64, 64, 3), np.uint8), 512, 0.5, 0.7, 2.3))      # before load
        asyncio.run(det.load("cuda:0"))
        page_a, page_b = synth.make_page(5, 512, 384, 6)[0], synth.make_page(4, 512, 512, 6)[0]
        strip = np.concatenate([synth.make_page(6 + i, 512, 256, 3)[0] for i in range(4)], axis=0)     # 2048 x 256: rearranged patches
        # (512x384 @512): pad path; (@768): host resize + pad path; (512x512 @512): device-resident path; the strip
        for page, detect_size in ((page_a, 512), (page_a, 768), (page_b, 512), (strip, 512)):
            lines, raw_mask, extra = asyncio.run(det.infer(page, detect_size, 0.5, 0.6, 2.3))
            r_lines, r_mask, _, _ = r34.detector_infer(sd, page, detect_size, 0.5, 0.6, 2.3)
            assert len(r_lines) > 5
            assert extra is None and raw_mask.dtype == np.uint8 and raw_mask.shape == r_mask.shape
            _assert_same_detections(lines, r_lines, raw_mask, r_mask)
        asyncio.run(det.unload())
    finally:
        plugins.DefaultDetector.set_state_dict(None)

"""TEST INFRASTRUCTURE -- oracle of the reference's default detector, DBNet-ResNet34 (detection/default.py, network
detection/default_utils/DBNet_resnet34.py): its seeded "hardened" state dict, a functional CPU fp32 restatement of the network
in the style of oracle/nets.py, and the `_infer` glue with this network behind it.  Pinned on the reference's own outputs
(tests/golden/reference_pins_default_detector.*, written by oracle/ref_pins_default_detector.py).  Nothing here is product code.

Layout: all tensors NCHW fp32 like the reference.
"""
from __future__ import annotations

from typing import Dict, Optional

import cv2
import numpy as np
import torch
import torch.nn.functional as F

from .weights import Spec, generate

from mit_b200.host import det_post, rearrange
from mit_b200.host.geometry import Quadrilateral

SD = Dict[str, torch.Tensor]
_BN_EPS = 1e-5                               # nn.BatchNorm2d default


# ----------------------------------------------------------------------------- seeded state dict
def _bn_spec(spec: Spec, p: str, c: int):
    spec += [(p + "weight", (c,), "bn_w"), (p + "bias", (c,), "bn_b"), (p + "running_mean", (c,), "bn_m"), (p + "running_var", (c,), "bn_v")]


def _conv_bn(spec: Spec, p: str, wname: str, bn: str, shape, kind="conv_act"):
    spec += [(p + wname, shape, kind)]
    _bn_spec(spec, p + bn, shape[1] if kind.startswith("convT") else shape[0])


def spec() -> Spec:
    """TextDetection().state_dict() (DBNet_resnet34.py:76-101), torchvision resnet34 backbone incl. fc; BN stats and affines hardened
    as in oracle/weights.py, the second conv of each BasicBlock drawn as a tamed residual branch."""
    s: Spec = []
    b = "backbone."
    _conv_bn(s, b, "conv1.weight", "bn1.", (64, 3, 7, 7))
    prev = 64
    for li, (blocks, c) in enumerate(((3, 64), (4, 128), (6, 256), (3, 512)), 1):
        for k in range(blocks):
            q = f"{b}layer{li}.{k}."
            cin = prev if k == 0 else c
            _conv_bn(s, q, "conv1.weight", "bn1.", (c, cin, 3, 3))
            _conv_bn(s, q, "conv2.weight", "bn2.", (c, c, 3, 3), "conv_res")     # residual branch of a post-activation block: tame
            if k == 0 and (li > 1):
                _conv_bn(s, q, "downsample.0.weight", "downsample.1.", (c, cin, 1, 1), "lin")
        prev = c
    s += [(b + "fc.weight", (1000, 512), "lin"), (b + "fc.bias", (1000,), "bias")]
    for br, bias in (("binarize", True), ("thresh", False)):
        p = f"conv_db.{br}."
        s += [(p + "0.weight", (16, 64, 3, 3), "conv_act")] + ([(p + "0.bias", (16,), "bias")] if bias else [])
        _bn_spec(s, p + "1.", 16)
        s += [(p + "3.weight", (16, 16, 4, 4), "convT4_act"), (p + "3.bias", (16,), "bias")]   # _init_upsample drops `bias`: both
        _bn_spec(s, p + "4.", 16)                                                              # branches' transposed convs have one
        s += [(p + "6.weight", (16, 1, 4, 4), "convT4_out"), (p + "6.bias", (1,), "bias")]
    for i, (cin, cout, k, kind) in enumerate(((64, 64, 3, "conv_act"), (64, 64, 3, "conv_act"), (64, 32, 3, "conv_act"), (32, 1, 1, "out"))):
        s += [(f"conv_mask.{2 * i}.weight", (cout, cin, k, k), kind), (f"conv_mask.{2 * i}.bias", (cout,), "bias")]
    for d in (1, 2, 3):
        p = f"down_conv{d}.conv."
        for j in (0, 3, 6):
            _conv_bn(s, p, f"{j}.weight", f"{j + 1}.", (512, 512, 3, 3))
    for u, (cin, mid, cout) in enumerate(((0, 512, 256), (256, 512, 256), (256, 512, 256), (256, 512, 256), (256, 256, 128),
                                          (128, 128, 64), (64, 64, 64)), 1):
        p = f"upconv{u}.conv."
        _conv_bn(s, p, "0.weight", "1.", (mid, cin + mid, 3, 3))
        _conv_bn(s, p, "3.weight", "4.", (mid, mid, 3, 3))
        _conv_bn(s, p, "6.weight", "7.", (mid, cout, 4, 4), "convT4_act")
    return s


def weights(seed: int = 1) -> SD:
    return generate(spec(), 5000 + seed)


# ----------------------------------------------------------------------------- network
def _bn(sd: SD, p: str, x):
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd[p + "weight"], sd[p + "bias"], False, 0.0, _BN_EPS)


def _block(sd: SD, p: str, x, stride: int):
    """torchvision BasicBlock.forward (post-activation): relu(bn2(conv2(relu(bn1(conv1 x)))) + identity)."""
    y = F.relu(_bn(sd, p + "bn1.", F.conv2d(x, sd[p + "conv1.weight"], stride=stride, padding=1)))
    y = _bn(sd, p + "bn2.", F.conv2d(y, sd[p + "conv2.weight"], padding=1))
    if p + "downsample.0.weight" in sd:
        x = _bn(sd, p + "downsample.1.", F.conv2d(x, sd[p + "downsample.0.weight"], stride=stride))
    return F.relu(y + x)


def _double_conv(sd: SD, p: str, x, up: bool):
    """double_conv (AvgPool2d(2,2) then three conv3x3+BN+ReLU, DBNet_resnet34.py:23-53) or double_conv_up (two conv3x3+BN+ReLU, then
    ConvTranspose2d(4, 2, 1, bias=False)+BN+ReLU, :55-74)."""
    if not up:
        x = F.avg_pool2d(x, 2, 2)
    x = F.relu(_bn(sd, p + "1.", F.conv2d(x, sd[p + "0.weight"], padding=1)))
    x = F.relu(_bn(sd, p + "4.", F.conv2d(x, sd[p + "3.weight"], padding=1)))
    if up:
        x = F.conv_transpose2d(x, sd[p + "6.weight"], stride=2, padding=1)
    else:
        x = F.conv2d(x, sd[p + "6.weight"], padding=1)
    return F.relu(_bn(sd, p + "7.", x))


def _db_head(sd: SD, x):
    """DBHead(64, 0).forward eval branch (default_utils/DBHead.py:7-34): binarize logits, sigmoid(thresh)."""
    def branch(q, final_sigmoid):
        y = F.relu(_bn(sd, q + "1.", F.conv2d(x, sd[q + "0.weight"], sd.get(q + "0.bias"), padding=1)))
        y = F.relu(_bn(sd, q + "4.", F.conv_transpose2d(y, sd[q + "3.weight"], sd.get(q + "3.bias"), stride=2, padding=1)))
        y = F.conv_transpose2d(y, sd[q + "6.weight"], sd.get(q + "6.bias"), stride=2, padding=1)
        return torch.sigmoid(y) if final_sigmoid else y
    return torch.cat([branch("conv_db.binarize.", False), branch("conv_db.thresh.", True)], dim=1)


def forward(sd: SD, x, taps: Optional[dict] = None):
    """TextDetection.forward (DBNet_resnet34.py:103-125) -> (db [N,2,H,W] before the caller's sigmoid, mask [N,1,H/2,W/2])."""
    b = "backbone."
    s = F.relu(_bn(sd, b + "bn1.", F.conv2d(x, sd[b + "conv1.weight"], stride=2, padding=3)))
    s = F.max_pool2d(s, 3, 2, 1)                        # -inf padding
    feats = []
    for li, blocks in enumerate((3, 4, 6, 3), 1):
        for k in range(blocks):
            s = _block(sd, f"{b}layer{li}.{k}.", s, 2 if (k == 0 and li > 1) else 1)
        feats.append(s)
    h4, h8, h16, h32 = feats
    h64 = _double_conv(sd, "down_conv1.conv.", h32, False)
    h128 = _double_conv(sd, "down_conv2.conv.", h64, False)
    h256 = _double_conv(sd, "down_conv3.conv.", h128, False)
    up256 = _double_conv(sd, "upconv1.conv.", h256, True)
    up128 = _double_conv(sd, "upconv2.conv.", torch.cat([up256, h128], 1), True)
    up64 = _double_conv(sd, "upconv3.conv.", torch.cat([up128, h64], 1), True)
    up32 = _double_conv(sd, "upconv4.conv.", torch.cat([up64, h32], 1), True)
    up16 = _double_conv(sd, "upconv5.conv.", torch.cat([up32, h16], 1), True)
    up8 = _double_conv(sd, "upconv6.conv.", torch.cat([up16, h8], 1), True)
    up4 = _double_conv(sd, "upconv7.conv.", torch.cat([up8, h4], 1), True)
    if taps is not None:
        taps.update(h4=h4, h8=h8, h16=h16, h32=h32, h64=h64, h128=h128, h256=h256, up8=up8, up4=up4)
    db = _db_head(sd, up8)
    m = up4
    for i in range(3):
        m = F.relu(F.conv2d(m, sd[f"conv_mask.{2 * i}.weight"], sd[f"conv_mask.{2 * i}.bias"], padding=1))
    m = torch.sigmoid(F.conv2d(m, sd["conv_mask.6.weight"], sd["conv_mask.6.bias"]))
    return db, m


def batch_forward(sd: SD, batch_u8_nhwc: np.ndarray):
    """det_batch_forward_default (detection/default.py:15-25): /127.5 - 1, forward, sigmoid on both db channels.  The input stays the
    NHWC-strided view that einops.rearrange hands the reference network (CPU convolutions then sum in the same order)."""
    x = batch_u8_nhwc.astype(np.float32) / 127.5 - 1.0
    x = torch.from_numpy(x.transpose(0, 3, 1, 2))
    db, mask = forward(sd, x)
    return db.sigmoid().numpy(), mask.numpy()


# ----------------------------------------------------------------------------- `_infer` glue
def detector_infer(sd, image: np.ndarray, detect_size: int, text_threshold: float, box_threshold: float, unclip_ratio: float):
    """DefaultDetector._infer (detection/default.py:56-103) on the host, fp32: line for line the DBConvNextDetector glue of
    oracle/pipeline_ref.detector_infer with this network behind it.  Returns (textlines, raw uint8 mask, db, mask)."""
    def fwd(batch):
        return batch_forward(sd, np.asarray(batch))

    db, mask = rearrange.rearrange_forward(image, fwd, detect_size, 4)
    if db is None:
        img_resized, ratio, _, pad_w, pad_h = det_post.resize_aspect_ratio(cv2.bilateralFilter(image, 17, 80, 80), detect_size,
                                                                          cv2.INTER_LINEAR, mag_ratio=1)
        rh, rw = img_resized.shape[:2]
        ratio_h = ratio_w = 1 / ratio
        db, mask = fwd([img_resized])
    else:
        rh, rw = image.shape[:2]
        ratio_w = ratio_h = 1
        pad_h = pad_w = 0
    mask = mask[0, 0]
    boxes, scores = det_post.boxes_from_prob(db[0, 0], text_threshold, box_threshold, unclip_ratio, rw, rh)
    polys = det_post.polys_from_boxes(boxes, scores, ratio_w, ratio_h)
    textlines = [Quadrilateral(p.astype(int), "", s) for p, s in zip(polys, scores)]
    textlines = [q for q in textlines if q.area > 16]
    up = cv2.resize(mask, (mask.shape[1] * 2, mask.shape[0] * 2), interpolation=cv2.INTER_LINEAR)
    if pad_h > 0:
        up = up[:-pad_h, :]
    elif pad_w > 0:
        up = up[:, :-pad_w]
    return textlines, np.clip(up * 255, 0, 255).astype(np.uint8), db, mask

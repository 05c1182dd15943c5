"""CPU: the oracle restatement of the default detector (DBNet-ResNet34, detection/default.py) against the reference's own outputs,
recorded by oracle/ref_pins_default_detector.py in tests/golden/reference_pins_default_detector.{json,npz}."""
import numpy as np
import torch

from oracle import cases, ref_pins
from oracle import dbnet_r34 as r34
from oracle import ref_pins_default_detector as pins


def _sampled(t):
    flat = t.numpy().reshape(-1)
    return flat[ref_pins.sample_positions(flat.size)]


def test_state_dict_spec_matches_reference():
    J, _ = pins.load()
    sd = r34.weights()
    assert ref_pins.state_dict_spec(sd) == J["state_dict_spec"]
    assert "backbone.fc.weight" in sd and "backbone.fc.bias" in sd


def test_network_matches_reference_at_two_sizes():
    J, Z = pins.load()
    sd = r34.weights(seed=2)
    with torch.no_grad():
        for h, w, n, seed in pins.NET_CASES:
            _, x = cases.dbnet_case(h, w, n=n, seed=seed)
            db, mask = r34.forward(sd, x)
            assert list(db.shape) == J[f"net_{h}x{w}_db_shape"] and list(mask.shape) == J[f"net_{h}x{w}_mask_shape"]
            assert np.abs(Z[f"net_{h}x{w}_db"] - _sampled(db)).max() < 1e-4
            assert np.abs(Z[f"net_{h}x{w}_mask"] - _sampled(mask)).max() < 1e-5


def test_default_detector_infer_glue_equals_reference_code():
    J, _ = pins.load()
    sd = pins.glue_weights()
    for (page, detect_size), want in zip(ref_pins.detector_glue_pages(), J["detector_glue"]):
        o_lines, o_mask, _, _ = r34.detector_infer(sd, page, detect_size, 0.5, 0.6, 2.3)
        assert len(want["lines"]) == len(o_lines) and len(o_lines) > 3
        for a, b in zip(want["lines"], o_lines):
            assert np.array_equal(np.array(a["pts"]), b.pts) and a["prob"] == b.prob and a["direction"] == b.direction
        assert want["mask_dtype"] == "uint8" and ref_pins.digest(o_mask) == want["mask"]


def test_fixture_is_the_oracle():
    """tests/golden/dbnet_r34_256x512.npz (read by the GPU tests) is what the pinned oracle computes."""
    z = np.load(pins.FIXTURE)
    _, x = pins.fixture_case()
    with torch.no_grad():
        db, mask = r34.forward(r34.weights(), x)
    assert np.abs(z["db_sigmoid"] - db.sigmoid().numpy()).max() < 1e-5 and np.abs(z["mask"] - mask.numpy()).max() < 1e-5

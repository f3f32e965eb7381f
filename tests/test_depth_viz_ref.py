"""The numpy restatement of visualize_depth (tests/depth_viz_ref.py) against what the unmodified reference returned
(tests/golden/depth_viz.npz, tests/golden/make_depth_viz_golden.py), bit for bit, and the committed JET table
against cv2 where cv2 is importable."""
import json
import os

import numpy as np
import pytest

from tests import depth_viz_ref as dv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "depth_viz.npz")
MAPS = ["trained", "nan", "posinf", "neginf", "negative", "constant", "one", "odd"]


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def test_fixture_holds_every_map(golden):
    meta = json.loads(str(golden["meta"]))
    assert meta["maps"] == MAPS
    assert golden["trained.depth"].shape == (200, 200)
    assert golden["one.depth"].shape == (1, 1) and golden["odd.depth"].shape == (37, 53)
    assert np.isnan(golden["nan.depth"]).any() and np.isposinf(golden["posinf.depth"]).any()
    assert np.isneginf(golden["neginf.depth"]).any() and (golden["negative.depth"] < 0).any()


@pytest.mark.parametrize("name", MAPS)
def test_restatement_equals_the_reference_bit_for_bit(golden, name):
    want = golden[f"{name}.out"]
    got = dv.visualize_depth(golden[f"{name}.depth"])
    assert got.dtype == np.float32 == want.dtype and got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_trained_map_uses_much_of_the_table(golden):
    u = dv.to_uint8(golden["trained.depth"])
    assert len(np.unique(u)) > 100 and u.min() == 0 and u.max() == 255


def test_channel_zero_is_blue():
    """The reference hands cv2's BGR array to Image.fromarray as RGB: the nearest depth (u8 0, JET dark blue) has
    channel 0 = 128 / 255 and the farthest (u8 255, dark red) has channel 2 = 128 / 255."""
    out = dv.visualize_depth(np.array([[1.0, 2.0]], np.float32))
    assert np.array_equal(out[:, 0, 0], np.float32([128, 0, 0]) / np.float32(255))
    assert np.array_equal(out[:, 0, 1], np.float32([0, 0, 128]) / np.float32(255))


def test_committed_table_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    want = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_JET)[:, 0, :]
    assert np.array_equal(dv.jet_lut(), want)
    head = open(dv.LUT_H).readline()
    assert "OpenCV" in head

"""The rotation edit on the host: parsing `model.rotation`, Rodrigues' formula, the identity rule, the ctypes arrays, the default
centre and the oriented default box of `layer_density` (stnerf_b200.rotation)."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import cases as C
from stnerf_b200 import _lib as L
from stnerf_b200 import rotation as ROT
from tests_support import make_cfg


def _model(rotation=None, L_=2):
    import modeling
    case = C.CASES["syn_L2_64_128"]
    model = modeling.build_layered_model(make_cfg(L_, 64, 128, True), 0, None, None, rotation=rotation)
    bkgd, frames = C.boxes_for(case)
    model.set_bkgd_bbox(bkgd)
    model.set_bboxes(frames)
    return model


@pytest.mark.parametrize("seed", range(6))
def test_rodrigues_matches_scipy(seed):
    v = np.random.RandomState(seed).normal(size=3) * (seed + 0.5)
    assert np.allclose(ROT.rodrigues(v), Rotation.from_rotvec(v).as_matrix(), atol=1e-13)
    R, c = ROT.parse_entry(v)
    assert R.dtype == np.float32 and c is None
    assert np.array_equal(R, Rotation.from_rotvec(v).as_matrix().astype(np.float32)) or \
        np.abs(R.astype(np.float64) - Rotation.from_rotvec(v).as_matrix()).max() <= 2 ** -24


def test_entry_forms():
    Rm = Rotation.from_rotvec([0.3, -0.2, 0.9]).as_matrix()
    R, c = ROT.parse_entry(Rm)
    assert np.array_equal(R, Rm.astype(np.float32)) and c is None
    R, c = ROT.parse_entry((Rm.tolist(), [1, 2, 3]))
    assert np.array_equal(c, np.float32([1, 2, 3])) and np.array_equal(R, Rm.astype(np.float32))
    R2, c2 = ROT.parse_entry(([0.3, -0.2, 0.9], (0.5, 0, -1)))
    assert np.array_equal(R2, ROT.rodrigues([0.3, -0.2, 0.9]).astype(np.float32)) and c2.dtype == np.float32
    assert ROT.parse_entry(None) is None


def test_identity_counts_as_none():
    assert ROT.parse_entry(np.eye(3)) is None
    assert ROT.parse_entry([0.0, 0.0, 0.0]) is None
    assert ROT.parse_entry((np.eye(3), [1, 2, 3])) is None
    assert ROT.resolve([None, np.eye(3), [0, 0, 0]], 3) == [None, None, None]
    modes, R, cen = ROT.abi_arrays([None, None, None])
    assert not modes.any()
    # nearly the identity is a rotation
    assert ROT.parse_entry([0, 0, 1e-6]) is not None


@pytest.mark.parametrize("bad", [np.diag([1.0, 1.0, -1.0]), 2 * np.eye(3), np.eye(3) + 1e-4, np.full((3, 3), np.nan),
                                 [np.inf, 0, 0], np.eye(4), [1.0, 2.0]])
def test_invalid_rotations_raise(bad):
    with pytest.raises(ValueError):
        ROT.parse_entry(bad)


def test_invalid_centre_raises():
    with pytest.raises(ValueError):
        ROT.parse_entry(([0, 0, 1], [0, np.nan, 0]))
    with pytest.raises(ValueError):
        ROT.parse_entry(([0, 0, 1], [0, 0]))


def test_short_list_raises_index_error_like_shift():
    with pytest.raises(IndexError):
        ROT.resolve([None, [0, 0, 1]], 3)
    model = _model(rotation=[None, [0, 0, 1]])
    with pytest.raises(IndexError):
        model._rotation_entries()


def test_abi_arrays():
    Rm = Rotation.from_rotvec([0, 0, 0.5]).as_matrix()
    modes, R, cen = ROT.abi_arrays(ROT.resolve([None, Rm, (Rm, [1, 2, 3])], 3))
    assert modes.tolist() == [L.ROT_OFF, L.ROT_BOX, L.ROT_CENTRE]
    assert R.dtype == np.float32 and R.shape == (3, 9) and np.array_equal(R[1], Rm.astype(np.float32).reshape(9))
    assert np.array_equal(cen[2], np.float32([1, 2, 3])) and not cen[1].any()


def test_constructor_and_mutable_attribute():
    Rm = Rotation.from_rotvec([0, 0, 0.5]).as_matrix()
    model = _model(rotation=[None, Rm, None])
    assert model._rotation_entries()[1] is not None
    model.rotation = None
    assert model._rotation_entries() == [None, None, None]


@pytest.mark.parametrize("frame", [10.0, 10.5])
def test_default_centre_is_the_edited_box_centre(frame):
    """The library's STNERF_ROT_BOX centre, (bmin + bmax) * 0.5 in fp32, equals the float64 centre rounded once."""
    model = _model()
    model.scale, model.shift = [1, 0.75, 1.5], [[0, 0, 0], [0, 0.3, 0], [0, -0.3, 0]]
    sc = model._resolve_scene(torch.full((3,), frame), 0.0, 0.0)
    for i in range(3):
        lo, hi = np.float64(sc.bmin[i][:]), np.float64(sc.bmax[i][:])
        assert np.array_equal(ROT.default_centre(sc.bmin[i][:], sc.bmax[i][:]), ((lo + hi) / 2).astype(np.float32))


@pytest.mark.parametrize("seed", range(4))
def test_oriented_box_aabb_against_float64(seed):
    rs = np.random.RandomState(seed)
    lo = rs.uniform(-2, 0, 3).astype(np.float32)
    hi = lo + rs.uniform(0.5, 2, 3).astype(np.float32)
    R = Rotation.from_rotvec(rs.normal(size=3)).as_matrix().astype(np.float32)
    c = rs.uniform(-1, 1, 3).astype(np.float32)
    mn, mx = ROT.oriented_box_aabb(lo, hi, R, c)
    corners = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float64)
    w = (R.astype(np.float64) @ (corners - c.astype(np.float64)).T).T + c.astype(np.float64)
    assert (np.float64(mn) <= w.min(0)).all() and (np.float64(mx) >= w.max(0)).all()
    # rounded outward by at most one float32 step
    assert (np.float64(mn) >= np.nextafter(w.min(0).astype(np.float32), np.float32(-np.inf)) - 1e-12).all()
    assert (np.float64(mx) <= np.nextafter(w.max(0).astype(np.float32), np.float32(np.inf)) + 1e-12).all()
    # a quarter turn about z of a box about its centre swaps the x and y extents exactly
    q = Rotation.from_rotvec([0, 0, np.pi / 2]).as_matrix().astype(np.float32)
    lo2, hi2 = np.float32([-1, -2, -3]), np.float32([1, 2, 3])
    mn, mx = ROT.oriented_box_aabb(lo2, hi2, q, np.zeros(3, np.float32))
    assert np.allclose(mn, [-2, -1, -3], atol=1e-6) and np.allclose(mx, [2, 1, 3], atol=1e-6)


def test_facade_signature_keeps_rotation_inert():
    import inspect
    from render import LayeredNeuralRenderer
    assert "rotation" in inspect.signature(LayeredNeuralRenderer.__init__).parameters
    assert hasattr(LayeredNeuralRenderer, "set_rotation")

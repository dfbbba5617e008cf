"""CPU: the surface-distance metric's host side — the derived surfel-area table against the reference's table, the
torch oracle against the reference's (ASD, HD) on the fixture cases, and the argument checks of calculate_distance."""
import os

import numpy as np
import pytest
import torch

import b200seg
from b200seg.surface import surface_area_table
from oracle import surface as osurf


@pytest.fixture(scope="module")
def tables(golden_dir):
    return torch.load(os.path.join(golden_dir, "surface_tables.pt"))


@pytest.fixture(scope="module")
def ref(golden_dir):
    return torch.load(os.path.join(golden_dir, "surface_ref.pt"))["cases"]


def _maps(case):
    dt = getattr(torch, case["dtype"].replace("torch.", ""))
    return case["pred"].to(dt), case["gt"].to(dt)


def test_table_matches_reference(tables):
    assert tables["spacings"].shape[0] >= 4
    for s, t in zip(tables["spacings"].tolist(), tables["tables"]):
        got = surface_area_table(s)
        t = t.numpy()
        assert got.shape == (256,)
        assert got[0] == 0 and got[255] == 0
        np.testing.assert_allclose(got, t, rtol=1e-12, atol=0, err_msg=str(s))


def test_table_accepts_tensor_and_array_spacing():
    a = surface_area_table((2.5, 0.78, 0.78))
    np.testing.assert_array_equal(surface_area_table(torch.tensor([2.5, 0.78, 0.78], dtype=torch.float64)), a)
    np.testing.assert_array_equal(surface_area_table(np.array([2.5, 0.78, 0.78])), a)
    with pytest.raises(ValueError):
        surface_area_table((1.0, 1.0))


def test_fixture_covers_the_edge_cases(ref):
    names = {c["name"] for c in ref}
    assert {"aniso", "faces", "single_voxel", "absent", "d1", "c16"} <= names
    assert {c["percentage"] for c in ref} >= {50, 95, 100}
    assert any(c["pred"].shape[0] == 1 for c in ref) and any(c["C"] == 16 for c in ref)
    assert {c["dtype"] for c in ref} == {"torch.int64", "torch.uint8"}


def test_oracle_reproduces_reference(ref):
    for c in ref:
        pred, gt = _maps(c)
        asd, hd = osurf.calculate_distance(pred, gt, c["spacing"], c["C"], percentage=c["percentage"])
        for got, want in ((asd, c["asd"].numpy()), (hd, c["hd"].numpy())):
            assert got.dtype == np.float64 and got.shape == (c["C"] - 1,)
            np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=c["name"])
            np.testing.assert_array_equal(np.isinf(got), np.isinf(want), err_msg=c["name"])
            fin = np.isfinite(want)
            np.testing.assert_allclose(got[fin], want[fin], rtol=1e-12, atol=0, err_msg=c["name"])


def test_calculate_distance_rejects_bad_ranks():
    v = torch.zeros(4, 5, 6, dtype=torch.int64)
    with pytest.raises(ValueError):
        b200seg.calculate_distance(v[None], v[None], [1, 1, 1], 3)
    with pytest.raises(ValueError):
        b200seg.calculate_distance(v[0], v[0], [1, 1, 1], 3)
    with pytest.raises(ValueError):
        b200seg.calculate_distance(v, v[:, :, :5], [1, 1, 1], 3)


def test_calculate_distance_has_no_cpu_fallback():
    v = torch.zeros(4, 5, 6, dtype=torch.int64)
    with pytest.raises(b200seg.B200SegError):
        b200seg.calculate_distance(v, v, [1, 1, 1], 3)

"""GPU: calculate_distance (csrc/surface.cu) against the reference's (ASD, HD) on the fixture cases and against the
brute-force torch oracle (oracle/surface.py) on validation-sized volumes; label dtypes, run-to-run bit equality."""
import os

import numpy as np
import pytest
import torch

import b200seg
from oracle import surface as osurf

pytestmark = pytest.mark.gpu


def _check(got, want, what, rtol=1e-9):
    assert got.dtype == np.float64 and got.shape == want.shape, what
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=what)
    np.testing.assert_array_equal(np.isinf(got), np.isinf(want), err_msg=what)
    fin = np.isfinite(want)
    np.testing.assert_allclose(got[fin], want[fin], rtol=rtol, atol=0, err_msg=what)


def test_fixture_cases_match_reference(golden_dir):
    cases = torch.load(os.path.join(golden_dir, "surface_ref.pt"))["cases"]
    for c in cases:
        dt = getattr(torch, c["dtype"].replace("torch.", ""))
        pred, gt = c["pred"].to(dt).cuda(), c["gt"].to(dt).cuda()
        asd, hd = b200seg.calculate_distance(pred, gt, torch.tensor(c["spacing"], dtype=torch.float64), c["C"], percentage=c["percentage"])
        _check(asd, c["asd"].numpy(), c["name"] + " ASD")
        _check(hd, c["hd"].numpy(), c["name"] + " HD")


@pytest.mark.parametrize("shape,C,spacing,pct", [((64, 160, 160), 4, (2.5, 0.78, 0.78), 95),
                                                  ((128, 256, 256), 3, (0.7, 1.3, 3.0), 95)])
def test_matches_oracle_at_validation_size(shape, C, spacing, pct):
    pred, gt = osurf.synthetic_pair(shape, C, seed=sum(shape) + C, device="cuda")
    want = osurf.calculate_distance(pred, gt, spacing, C, percentage=pct)
    got = b200seg.calculate_distance(pred, gt, np.array(spacing), C, percentage=pct)
    _check(got[0], want[0], "ASD %s" % (shape,))
    _check(got[1], want[1], "HD %s" % (shape,))


def test_label_dtypes_and_run_to_run_bits():
    pred, gt = osurf.synthetic_pair((40, 72, 64), 5, seed=3, device="cuda")
    sp = [1.0, 1.0, 5.0]
    base = b200seg.calculate_distance(pred, gt, sp, 5, percentage=95)
    again = b200seg.calculate_distance(pred, gt, sp, 5, percentage=95)
    for a, b in zip(base, again):
        assert a.tobytes() == b.tobytes()
    for p, g in ((pred.to(torch.uint8), gt.to(torch.uint8)), (pred.to(torch.uint8), gt), (pred, gt.to(torch.uint8)),
                 (pred.int(), gt.short())):
        out = b200seg.calculate_distance(p, g, sp, 5, percentage=95)
        for a, b in zip(base, out):
            assert a.tobytes() == b.tobytes()
    want = osurf.calculate_distance(pred, gt, sp, 5, percentage=95)
    _check(base[0], want[0], "ASD")
    _check(base[1], want[1], "HD")


def test_non_contiguous_maps_and_out_of_range_labels():
    pred, gt = osurf.synthetic_pair((24, 48, 40), 4, seed=9, device="cuda")
    gt[0, 0, :5] = 7                        # labels >= C belong to no class, as label == c in the reference
    pt = pred.transpose(1, 2).contiguous().transpose(1, 2)
    got = b200seg.calculate_distance(pt, gt, [2.0, 1.0, 1.0], 4, percentage=90)
    want = osurf.calculate_distance(pred, gt, [2.0, 1.0, 1.0], 4, percentage=90)
    _check(got[0], want[0], "ASD")
    _check(got[1], want[1], "HD")


def test_cpu_tensors_raise():
    pred, gt = osurf.synthetic_pair((8, 8, 8), 3, seed=1)
    with pytest.raises(b200seg.B200SegError):
        b200seg.calculate_distance(pred, gt, [1, 1, 1], 3)

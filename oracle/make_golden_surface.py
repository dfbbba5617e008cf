"""Pin the surface-distance metric to the UNMODIFIED reference (metric/utils.py:8-28 calculate_distance,
metric/lookup_tables.py create_table_neighbour_code_to_surface_area) and write
  tests/golden/surface_tables.pt  the reference's 256-entry surfel-area table at several spacings;
  tests/golden/surface_ref.pt     small seeded label-map pairs with the reference's (ASD_list, HD_list).
It also checks that oracle/surface.py reproduces the reference on every case.  Runs only where the reference
checkout exists.  Usage:  python oracle/make_golden_surface.py

Shims, applied before the reference is imported (the reference itself is not modified):
  * np.Inf = np.inf  — the reference pins numpy < 2 and returns np.Inf for an empty mask; numpy 2 removed the alias;
  * scipy.ndimage.filters / .morphology are the deprecated aliases the reference calls; they are used as they are."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_golden import REF          # noqa: E402

SPACINGS = [(1.0, 1.0, 1.0), (2.5, 0.78, 0.78), (0.7, 1.3, 3.0), (1.0, 1.0, 5.0), (3.0, 0.5, 0.5)]


def blobs(shape, C, seed, scale=3.0, keep=None):
    """Seeded label map [D,H,W] int64 in 0..C-1: smoothed noise, thresholded per class."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(C, *shape, generator=g, dtype=torch.float64)
    k = max(1, int(scale))
    ks = [2 * k + 1 if n > 2 * k else 1 for n in shape]
    x = torch.nn.functional.avg_pool3d(x[None], ks, stride=1, padding=[q // 2 for q in ks], count_include_pad=False)[0]
    x[0] += 0.15                         # a little more background
    lab = x.argmax(0)
    if keep is not None:
        lab[~torch.isin(lab, torch.tensor(keep))] = 0
    return lab


def cases():
    out = []
    # anisotropic spacing, 3 classes
    out.append(dict(name="aniso", pred=blobs((12, 20, 24), 3, 1), gt=blobs((12, 20, 24), 3, 2),
                    spacing=(2.5, 0.78, 0.78), C=3, percentage=95))
    # objects touching every face of the volume
    g = torch.ones(9, 11, 13, dtype=torch.int64)
    g[3:6, 4:7, 5:8] = 2
    p = torch.ones(9, 11, 13, dtype=torch.int64)
    p[0, :, :] = 0
    p[2:7, 3:8, 4:10] = 2
    out.append(dict(name="faces", pred=p, gt=g, spacing=(0.7, 1.3, 3.0), C=3, percentage=95))
    # single-voxel objects
    g = torch.zeros(8, 9, 10, dtype=torch.int64)
    p = torch.zeros(8, 9, 10, dtype=torch.int64)
    g[0, 0, 0] = 1; g[7, 8, 9] = 1; g[4, 4, 4] = 2
    p[1, 0, 0] = 1; p[3, 5, 6] = 2; p[0, 8, 0] = 2
    out.append(dict(name="single_voxel", pred=p, gt=g, spacing=(1.0, 1.0, 1.0), C=3, percentage=95))
    # class 1 absent from pred, class 2 absent from gt, class 3 absent from both
    g = blobs((10, 14, 12), 3, 3, keep=[1])
    p = blobs((10, 14, 12), 3, 4, keep=[2])
    out.append(dict(name="absent", pred=p, gt=g, spacing=(1.0, 1.0, 5.0), C=4, percentage=95))
    # a single slice
    out.append(dict(name="d1", pred=blobs((1, 24, 20), 3, 5), gt=blobs((1, 24, 20), 3, 6),
                    spacing=(2.5, 0.78, 0.78), C=3, percentage=95))
    # percentiles
    for i, pc in enumerate((50, 100)):
        out.append(dict(name="perc%d" % pc, pred=blobs((14, 16, 18), 3, 7 + i), gt=blobs((14, 16, 18), 3, 9 + i),
                        spacing=(3.0, 0.5, 0.5), C=3, percentage=pc))
    # identical-area surfels with the boundary on percent / 100: a cube against a shifted cube, isotropic spacing
    g = torch.zeros(12, 12, 12, dtype=torch.int64)
    p = torch.zeros(12, 12, 12, dtype=torch.int64)
    g[2:8, 2:8, 2:8] = 1
    p[3:9, 2:8, 2:8] = 1
    out.append(dict(name="cube50", pred=p, gt=g, spacing=(1.0, 1.0, 1.0), C=2, percentage=50))
    # 16 classes (AMOS)
    out.append(dict(name="c16", pred=blobs((16, 24, 24), 16, 11, scale=2), gt=blobs((16, 24, 24), 16, 12, scale=2),
                    spacing=(2.5, 0.78, 0.78), C=16, percentage=95))
    # uint8 maps, the dtype inference_sliding_window(return_label=True) produces
    out.append(dict(name="uint8", pred=blobs((10, 18, 16), 4, 13).to(torch.uint8), gt=blobs((10, 18, 16), 4, 14).to(torch.uint8),
                    spacing=(1.0, 1.0, 1.0), C=4, percentage=95))
    return out


def main():
    np.Inf = np.inf                      # see the module docstring
    sys.path.insert(0, REF)
    import metric.utils as ref_utils
    from metric import lookup_tables
    from oracle import surface as osurf
    tables = {"spacings": torch.tensor(SPACINGS, dtype=torch.float64),
              "tables": torch.stack([torch.from_numpy(lookup_tables.create_table_neighbour_code_to_surface_area(s))
                                     for s in SPACINGS])}
    ref = []
    for c in cases():
        asd, hd = ref_utils.calculate_distance(c["pred"], c["gt"], torch.tensor(c["spacing"], dtype=torch.float64), c["C"],
                                               percentage=c["percentage"])
        oasd, ohd = osurf.calculate_distance(c["pred"], c["gt"], c["spacing"], c["C"], percentage=c["percentage"])
        for name, r, o in (("ASD", asd, oasd), ("HD", hd, ohd)):
            assert np.array_equal(np.isnan(r), np.isnan(o)) and np.array_equal(np.isinf(r), np.isinf(o)), (c["name"], name, r, o)
            fin = np.isfinite(r)
            assert np.allclose(r[fin], o[fin], rtol=1e-12, atol=0), (c["name"], name, r, o)
        print("%-12s C=%2d p=%3d  ASD %s  HD %s" % (c["name"], c["C"], c["percentage"], np.round(asd, 4), np.round(hd, 4)))
        # maps stored as uint8 (all labels < 256); "dtype" is the dtype the case runs with
        ref.append(dict(c, pred=c["pred"].to(torch.uint8), gt=c["gt"].to(torch.uint8), dtype=str(c["pred"].dtype),
                        asd=torch.from_numpy(asd), hd=torch.from_numpy(hd)))
    gold = os.path.join(ROOT, "tests", "golden")
    torch.save(tables, os.path.join(gold, "surface_tables.pt"))
    torch.save({"cases": ref}, os.path.join(gold, "surface_ref.pt"))
    print("wrote surface_tables.pt, surface_ref.pt")


if __name__ == "__main__":
    main()

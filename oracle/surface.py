"""Torch-only restatement of the reference's calculate_distance (metric/utils.py:8-28, metric/metrics.py:265-720).

Independent of csrc/surface.cu: the nearest-border distances are found by brute force over all border pairs (chunked,
fp64, scipy's formula sqrt(((Δ0·s0)² + (Δ1·s1)²) + (Δ2·s2)²) on integer offsets), the neighbour codes by shifted
slices of the whole grid, and the sums / percentile with numpy exactly as the reference writes them.  Needs no
scipy, so it runs wherever torch does (CUDA tensors keep the pair search on the GPU).  The surfel-area table is
b200seg.surface.surface_area_table, pinned separately to the reference's table."""
import numpy as np
import torch

from b200seg.surface import surface_area_table


def synthetic_pair(shape, C, seed, device="cpu"):
    """Seeded organ-like (pred, gt) int64 label maps: per foreground class one to three ellipsoids in gt, and the same
    ellipsoids shifted by up to 3 voxels and rescaled by up to 15 % in pred (later classes overwrite earlier ones)."""
    g = torch.Generator().manual_seed(seed)
    grid = torch.stack(torch.meshgrid(*[torch.arange(n, dtype=torch.float32) for n in shape], indexing="ij"))
    gt = torch.zeros(shape, dtype=torch.int64)
    pred = torch.zeros(shape, dtype=torch.int64)
    for c in range(1, C):
        for _ in range(int(torch.randint(1, 4, (1,), generator=g))):
            ctr = torch.rand(3, generator=g) * torch.tensor(shape, dtype=torch.float32)
            rad = (0.04 + 0.12 * torch.rand(3, generator=g)) * torch.tensor(shape, dtype=torch.float32) + 1.0
            shift = torch.randint(-3, 4, (3,), generator=g).float()
            scale = 0.85 + 0.3 * torch.rand(3, generator=g)
            for lab, cc, rr in ((gt, ctr, rad), (pred, ctr + shift, rad * scale)):
                inside = ((((grid - cc[:, None, None, None]) / rr[:, None, None, None]) ** 2).sum(0)) <= 1.0
                lab[inside] = c
    return pred.to(device), gt.to(device)


def neighbour_codes(mask):
    """uint8 codes on the grid extended by one voxel at the high end of each axis; bit 2**(7-(4a+2b+c)) is the voxel
    at offset (a-1, b-1, c-1), voxels outside the volume count as 0."""
    D, H, W = mask.shape
    m = torch.zeros(D + 2, H + 2, W + 2, dtype=torch.int32, device=mask.device)
    m[1:D + 1, 1:H + 1, 1:W + 1] = mask.to(torch.int32)
    code = torch.zeros(D + 1, H + 1, W + 1, dtype=torch.int32, device=mask.device)
    for k in range(8):
        a, b, c = k >> 2, (k >> 1) & 1, k & 1
        code |= m[a:a + D + 1, b:b + H + 1, c:c + W + 1] << (7 - k)
    return code


def _nearest(src, dst, spacing, chunk):
    """fp64 distance from every point of src [n,3] (int64) to the nearest point of dst [m,3]; inf if dst is empty."""
    if dst.shape[0] == 0:
        return torch.full((src.shape[0],), float("inf"), dtype=torch.float64, device=src.device)
    sp = torch.tensor(spacing, dtype=torch.float64, device=src.device)
    out = torch.empty(src.shape[0], dtype=torch.float64, device=src.device)
    for i in range(0, src.shape[0], chunk):
        s = src[i:i + chunk]
        best = torch.full((s.shape[0],), float("inf"), dtype=torch.float64, device=src.device)
        for j in range(0, dst.shape[0], chunk):
            d = (dst[None, j:j + chunk, :] - s[:, None, :]).to(torch.float64) * sp
            d = d * d
            d2 = (d[..., 0] + d[..., 1]) + d[..., 2]
            best = torch.minimum(best, d2.min(1).values)
        out[i:i + s.shape[0]] = best.sqrt()
    return out


def surface_distances(gt, pred, spacing, chunk=2048):
    """compute_surface_distances: (dist gt->pred, areas gt, dist pred->gt, areas pred), each sorted by (dist, area)."""
    table = torch.from_numpy(surface_area_table(spacing)).to(gt.device)
    cg, cp = neighbour_codes(gt), neighbour_codes(pred)
    bg = (cg != 0) & (cg != 255)
    bp = (cp != 0) & (cp != 255)
    pg, pp = bg.nonzero(), bp.nonzero()
    d_gp = _nearest(pg, pp, spacing, chunk)
    d_pg = _nearest(pp, pg, spacing, chunk)
    res = []
    for d, code, border in ((d_gp, cg, bg), (d_pg, cp, bp)):
        d = d.cpu().numpy()
        a = table[code[border].long()].cpu().numpy()
        order = np.lexsort((a, d))
        res += [d[order], a[order]]
    return res


def calculate_distance(label_pred, label_true, spacing, C, percentage=95):
    """(ASD_list, HD_list) numpy float64 [C-1] with the reference's formulas, nan / inf for missing classes."""
    spacing = [float(s) for s in (spacing.tolist() if hasattr(spacing, "tolist") else spacing)]
    asd, hd = np.zeros(C - 1), np.zeros(C - 1)
    for i in range(C - 1):
        gt, pred = label_true == i + 1, label_pred == i + 1
        if not bool((gt | pred).any()):
            d_gp = a_gp = d_pg = a_pg = np.zeros(0)
        else:
            d_gp, a_gp, d_pg, a_pg = surface_distances(gt, pred, spacing)
        with np.errstate(invalid="ignore", divide="ignore"):
            asd[i] = (np.sum(d_gp * a_gp) / np.sum(a_gp) + np.sum(d_pg * a_pg) / np.sum(a_pg)) / 2
        perc = []
        for d, a in ((d_gp, a_gp), (d_pg, a_pg)):
            if len(d) == 0:
                perc.append(np.inf)
                continue
            idx = np.searchsorted(np.cumsum(a) / np.sum(a), percentage / 100.0)
            perc.append(d[min(idx, len(d) - 1)])
        hd[i] = max(perc[0], perc[1])
    return asd, hd

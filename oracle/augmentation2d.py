"""TEST INFRASTRUCTURE — numpy float64 restatement of the reference's 2D augmentation (training/augmentation.py, the
2D branches) and of the ACDC slice branch (training/dataset/dim2/dataset_acdc.py:128-142), with every random quantity
passed in explicitly.  Pinned against the unmodified reference by oracle/make_golden_augmentation2d.py
(tests/golden/augment2d_*.pt).  Nothing in the product imports this file.

Array conventions: image [C, H, W]; label integer [H, W]."""
import math

import numpy as np
import torch
import torch.nn.functional as F


def make_slice(H, W, classes, seed):
    """A smooth synthetic MR-like slice (values ~[0, 1.5]) and a blob label map with every class present."""
    g = torch.Generator().manual_seed(seed)
    lo = (max(2, H // 12), max(2, W // 12))
    field = F.interpolate(torch.randn(1, 1, *lo, generator=g), size=(H, W), mode="bicubic", align_corners=True)
    img = (0.6 + 0.3 * field + 0.01 * torch.randn(1, 1, H, W, generator=g)).clamp(0.0, 1.5)
    lf = torch.randn(1, classes, *lo, generator=g)
    lf[:, 0] += 1.0
    lab = F.interpolate(lf, size=(H, W), mode="bilinear", align_corners=True).argmax(1)[0]
    flat = lab.view(-1)
    for c in range(classes):
        flat[c] = c
    return img[0, 0].float().contiguous(), lab.to(torch.uint8).contiguous()


# ---- geometry -------------------------------------------------------------------------------------------------------
def theta_from_draws(r6, angle_deg):
    """The 2x3 matrix of augmentation.py:200-214 from its seven random numbers (r6 = the six np.random.random() draws
    already mapped to sx, sy, shx, shy, tx, ty), in float32 like the reference's torch.mm."""
    sx, sy, hx, hy, tx, ty = r6
    S = torch.tensor([[sx, hx, tx], [hy, sy, ty], [0, 0, 1]]).float()
    a = (float(angle_deg) / 180.) * math.pi
    R = torch.tensor([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]]).float()
    return torch.mm(S, R)[0:2, :].numpy()


def draws_affine_2d(scale, rotate, translate):
    """The seven numpy draws of random_scale_rotate_translate_2d, in the reference's order."""
    s, t = float(scale), float(translate)
    sx = 1 - s + np.random.random() * 2 * s
    sy = 1 - s + np.random.random() * 2 * s
    hx = np.random.random() * 2 * s - s
    hy = np.random.random() * 2 * s - s
    tx = np.random.random() * 2 * t - t
    ty = np.random.random() * 2 * t - t
    ang = float(np.random.randint(-rotate, max(rotate, 1)))
    return (sx, sy, hx, hy, tx, ty), ang


def affine_grid(theta, H, W):
    """F.affine_grid(theta[None], (1, C, H, W), align_corners=True): base (linspace(-1, 1, W), linspace(-1, 1, H), 1)
    times theta^T, channels (x, y); float64."""
    th = np.asarray(theta, dtype=np.float64).reshape(2, 3)

    def lin(n):
        return np.linspace(-1.0, 1.0, n) if n > 1 else np.zeros(1)
    y, x = np.meshgrid(lin(H), lin(W), indexing="ij")
    base = np.stack([x, y, np.ones_like(x)], axis=-1)               # [H, W, 3]
    return base @ th.T                                              # [H, W, 2]


def grid_sample(img, grid, mode):
    """F.grid_sample(img[None], grid[None], mode, padding_mode='zeros', align_corners=True) in float64.
    img [C, H, W]; mode 'bilinear' or 'nearest' (round half to even)."""
    C, H, W = img.shape
    img = np.asarray(img, dtype=np.float64)
    ix = (grid[..., 0] + 1) * 0.5 * (W - 1)
    iy = (grid[..., 1] + 1) * 0.5 * (H - 1)

    def fetch(yi, xi):
        ok = (yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)
        v = img[:, np.clip(yi, 0, H - 1), np.clip(xi, 0, W - 1)]
        return np.where(ok[None], v, 0.0)
    if mode == "nearest":
        return fetch(np.rint(iy).astype(np.int64), np.rint(ix).astype(np.int64))
    x0, y0 = np.floor(ix), np.floor(iy)
    tx, ty = ix - x0, iy - y0
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    out = np.zeros((C,) + grid.shape[:2])
    for dy in (0, 1):
        for dx in (0, 1):
            w = (tx if dx else 1 - tx) * (ty if dy else 1 - ty)
            out += fetch(y0 + dy, x0 + dx) * w[None]
    return out


def scale_rotate_translate_2d(img, lab, theta):
    """random_scale_rotate_translate_2d (augmentation.py:192-223) for a given 2x3 theta."""
    grid = affine_grid(theta, *img.shape[1:])
    out = grid_sample(img, grid, "bilinear")
    olab = None if lab is None else grid_sample(np.asarray(lab, np.float64)[None], grid, "nearest")[0].astype(np.int64)
    return out, olab


def crop_2d(img, lab, origin, size):
    """crop_2d slicing (augmentation.py:313-314)."""
    y, x = origin
    h, w = size
    return img[:, y:y + h, x:x + w].copy(), None if lab is None else lab[y:y + h, x:x + w].copy()


# ---- intensity ------------------------------------------------------------------------------------------------------
def gamma(img, g, retain_stats=True):
    """augmentation.py:104-137 on one statistics row, float64 (std unbiased)."""
    x = np.asarray(img, dtype=np.float64).reshape(-1)
    mn, mx = x.min(), x.max()
    rng = mx - mn
    mean, std = x.mean(), x.std(ddof=1)
    y = np.power((x - mn) / rng, float(g)) * rng + mn
    if retain_stats:
        y = (y - y.mean()) / y.std(ddof=1) * std + mean
    return y.reshape(np.shape(img))


def contrast(img, f, preserve_range=True):
    """augmentation.py:139-173, float64."""
    x = np.asarray(img, dtype=np.float64).reshape(-1)
    mn, mx, mean = x.min(), x.max(), x.mean()
    y = (x - mean) * float(f) + mean
    if preserve_range:
        y = np.clip(y, mn, mx)
    return y.reshape(np.shape(img))


def gaussian_blur(img, sigma):
    """gaussian_blur on [C, H, W] (augmentation.py:46-64, the 2D branch): cross-correlation with the normalised dense
    k x k Gaussian, zero padding k//2, k = 2*ceil(3 sigma)+1; float64."""
    from scipy import ndimage
    k = 2 * math.ceil(3 * sigma) + 1
    r = np.arange(-k // 2 + 1, k // 2 + 1, dtype=np.float64)
    yy, xx = np.meshgrid(r, r, indexing="ij")
    ker = np.exp(-(xx ** 2 + yy ** 2) / (2 * sigma ** 2))
    ker /= ker.sum()
    return np.stack([ndimage.correlate(np.asarray(c, np.float64), ker, mode="constant", cval=0.0) for c in img])


# ---- the ACDC slice branch for given parameters -----------------------------------------------------------------------
def train_branch(noisy, lab, beta, g, theta, crop, size):
    """dataset_acdc.py:128-142 for one slice.  noisy: [H, W], the image after gaussian_noise (the noise is random by
    construction, so the caller supplies the noisy image); then brightness_additive (beta), gamma(g, retain_stats),
    the affine with theta over the whole slice and crop_2d at `crop` of extent `size`.  Returns ([h, w], [h, w]).
    The brightness output is rounded to float32, the tensor the reference hands to gamma: with gamma < 1 the power's
    slope is unbounded at the slice minimum, so the rounding of its input is part of the result."""
    y1 = (np.asarray(noisy, dtype=np.float32)[None] + np.float32(beta)).astype(np.float64)
    y3 = gamma(y1, g)
    i, l = scale_rotate_translate_2d(y3, lab, theta)
    i, l = crop_2d(i, l, crop, size)
    return i[0], l


def branch_coordinate_slack(noisy, beta, g, theta, crop, size, ulps=2):
    """How far the branch's image may move when its sampling positions move by `ulps` float32 ulps of the slice extent
    (both axes, all four sign combinations): [h, w].  The reference computes the positions in float32, so any
    float32 implementation is only defined to that precision, and a steep neighbourhood turns it into a visible
    difference (~1e-4 at 400 px with gamma 1.5)."""
    y1 = (np.asarray(noisy, dtype=np.float32)[None] + np.float32(beta)).astype(np.float64)
    y3 = gamma(y1, g)
    H, W = y3.shape[1:]
    y0, x0 = crop
    grid = affine_grid(theta, H, W)[y0:y0 + size[0], x0:x0 + size[1]]
    base = grid_sample(y3, grid, "bilinear")[0]
    eps = ulps * 2.0 ** -23 * max(H, W)
    slack = np.zeros_like(base)
    for sx in (-1, 1):
        for sy in (-1, 1):
            d = np.array([sx * eps * 2 / max(W - 1, 1), sy * eps * 2 / max(H - 1, 1)])
            slack = np.maximum(slack, np.abs(grid_sample(y3, grid + d, "bilinear")[0] - base))
    return slack

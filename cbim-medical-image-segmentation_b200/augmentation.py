"""GPU augmentation on the H100 (SURVEY.md §8f.3) behind the reference's ``training/augmentation.py`` interface.

The reference's ``aug_device: gpu`` path runs every augmentation as a chain of stock PyTorch ops per sample
(``training/dataset/dim3/dataset_kits.py:116-153``): slice + ``.contiguous()``, ``F.affine_grid`` + two
``F.grid_sample`` over a (size+60)^3 sub-volume, a second crop, three ``torch.flip`` copies, min/max/mean/std reductions
per intensity op, a dense 5^3/7^3 ``F.conv3d`` blur and a host-generated noise volume copied to the device.  Here:

  * every function of that module has a same-named counterpart with the same signature, the same random draws (same
    generators, same order — seeding ``numpy``/``torch`` reproduces the reference's decisions) and kernels from
    ``csrc/augment.cu`` instead of library calls;
  * :class:`TrainAugment3D` is the whole training branch as a *plan + 2..7 launches*: all random numbers are drawn first
    (they never depend on data), then ONE gather produces the final patch (crop -> affine -> centre crop -> mirrors), and
    each intensity op reads the statistics its predecessor left on the device — no reduction passes, no host sync;
  * :class:`TrainAugment2D` is the 2D (ACDC) slice branch for a whole batch of ragged slices in three launches
    (``b200seg_aug2d_train``), writing the ``[B, 1, h, w]`` batch the 2D models and losses take.

Images are ``[1, C, D, H, W]`` (volumes) or ``[1, C, H, W]`` (slices) fp32 CUDA tensors, label maps ``[1, 1, D, H, W]``
or ``[1, 1, H, W]`` uint8 or int64.  The 2D geometry runs on the 3D gather with D = 1.  There is no CPU path."""
import math
import struct

import numpy as np
import torch

from ._lib import B200SegError, call
from ._lib import load as load_lib
from .ops import _need_cuda, _stream

OP_MUL, OP_ADD, OP_GAMMA_POW, OP_RENORM, OP_CONTRAST, OP_NOISE, OP_STATS = range(7)

_I3 = torch.int32


# ----------------------------------------------------------------------------- device statistics rows
_STAT_TEMPLATES = {}


def new_stats(rows, device):
    """[rows, 4] int64 = {min key, max key, sum (double bits), sumsq (double bits)} initialised empty (include/b200seg.h)."""
    key = (rows, str(device))
    t = _STAT_TEMPLATES.get(key)
    if t is None:
        t = torch.tensor([[0xFFFFFFFF, 0, 0, 0]] * rows, dtype=torch.int64).to(device)
        _STAT_TEMPLATES[key] = t
    return t.clone()


def decode_stats(stats, n):
    """Host view of a statistics tensor: dict of per-row min / max / mean / std (unbiased).  Synchronises — tests only."""
    s = stats.cpu()
    keys = s[:, :2].numpy().astype(np.uint64).astype(np.uint32)
    bits = np.where(keys & np.uint32(0x80000000), keys & np.uint32(0x7FFFFFFF), ~keys).astype(np.uint32)
    mnmx = bits.view(np.float32)
    sums = s[:, 2:].contiguous().view(torch.float64).numpy()
    mean = sums[:, 0] / n
    var = (sums[:, 1] - n * mean * mean) / max(n - 1, 1)
    return {"min": mnmx[:, 0], "max": mnmx[:, 1], "mean": mean, "std": np.sqrt(np.maximum(var, 0))}


def _img(t):
    _need_cuda(t)
    if t.dim() not in (4, 5) or t.shape[0] != 1:
        raise ValueError("expected a [1, C, D, H, W] volume or a [1, C, H, W] image")
    if t.dtype != torch.float32:
        raise TypeError("images are fp32 (the reference augments before autocast), got %s" % t.dtype)
    return t.contiguous()


def _vol(*ts):
    """The volume functions take [1, C, D, H, W] tensors only: a [1, C, H, W] slice would hand the gather two-element
    geometry arrays where it reads three (the 2D functions make the [1, C, 1, H, W] view themselves)."""
    for t in ts:
        if t is not None and t.dim() != 5:
            raise ValueError("expected a [1, C, D, H, W] volume, got %s (use the 2D functions for slices)" % list(t.shape))


def _lab(t):
    _need_cuda(t)
    if t.dtype not in (torch.uint8, torch.int64):
        t = t.long()
    return t.contiguous()


def _rows(C, per_channel):
    return C if per_channel else 1


def _host_f(vals):
    return (torch.as_tensor(vals, dtype=torch.float32).reshape(-1).contiguous())


def _pointwise(x, op, a=None, b=None, rows=1, stats_in=None, stats_in2=None, want_stats=False, seed=0, out=True):
    x = _img(x)
    n = x.numel() // rows
    y = torch.empty_like(x) if out else None
    so = new_stats(rows, x.device) if want_stats else None
    ah = None if a is None else _host_f(a)
    bh = None if b is None else _host_f(b)
    call("b200seg_aug_pointwise", x.data_ptr(), None if y is None else y.data_ptr(), rows, n, op,
         None if ah is None else ah.data_ptr(), None if bh is None else bh.data_ptr(),
         None if stats_in is None else stats_in.data_ptr(), None if stats_in2 is None else stats_in2.data_ptr(),
         None if so is None else so.data_ptr(), int(seed) & 0xFFFFFFFFFFFFFFFF, _stream())
    return y, so


def image_stats(tensor_img, per_channel=False):
    """{min, max, sum, sum^2} of an image as a device statistics tensor (one pass)."""
    rows = _rows(tensor_img.shape[1], per_channel)
    return _pointwise(tensor_img, OP_STATS, rows=rows, want_stats=True, out=False)[1]


# ----------------------------------------------------------------------------- geometry
def resample(tensor_img, tensor_lab, sub_origin, sub_size, theta, out_origin, out_size, flips=(False, False, False),
             want_stats=False, per_channel=False, out_label_dtype=torch.int64):
    """The fused gather (``b200seg_aug_resample``).  theta: [3,4] float tensor / array (affine branch) or None (copy)."""
    _vol(tensor_img, tensor_lab)
    if any(len(v) != 3 for v in (sub_origin, sub_size, out_origin, out_size, flips)):
        raise ValueError("origins, sizes and flips of the volume gather have three entries (D, H, W)")
    img = None if tensor_img is None else _img(tensor_img)
    lab = None if tensor_lab is None else _lab(tensor_lab)
    ref = img if img is not None else lab
    C = 0 if img is None else img.shape[1]
    src = torch.tensor(list(ref.shape[2:]), dtype=_I3)
    so, ss = torch.tensor(list(sub_origin), dtype=_I3), torch.tensor(list(sub_size), dtype=_I3)
    oo, os_ = torch.tensor(list(out_origin), dtype=_I3), torch.tensor(list(out_size), dtype=_I3)
    th = None if theta is None else torch.as_tensor(theta, dtype=torch.float32).reshape(12).contiguous()
    out_img = None if img is None else torch.empty(1, C, *out_size, dtype=torch.float32, device=ref.device)
    out_lab = None if lab is None else torch.empty(1, 1, *out_size, dtype=out_label_dtype, device=ref.device)
    rows = _rows(C, per_channel)
    st = new_stats(rows, ref.device) if want_stats else None
    mask = (1 if flips[0] else 0) | (2 if flips[1] else 0) | (4 if flips[2] else 0)
    call("b200seg_aug_resample", None if img is None else img.data_ptr(), None if lab is None else lab.data_ptr(),
         0 if lab is None else lab.element_size(), C, src.data_ptr(), so.data_ptr(), ss.data_ptr(),
         None if th is None else th.data_ptr(), oo.data_ptr(), os_.data_ptr(), mask,
         None if out_img is None else out_img.data_ptr(),
         None if out_lab is None else out_lab.data_ptr(), 0 if out_lab is None else out_lab.element_size(),
         None if st is None else st.data_ptr(), rows, _stream())
    return out_img, out_lab, st


def _triple(v):
    return [v] * 3 if isinstance(v, (int, float)) else list(v)


def draw_affine_theta(scale=0.3, rotate=45, translate=0.1, shear=0.05):
    """The random 3x4 matrix of ``random_scale_rotate_translate_3d`` (augmentation.py:226-286): same numpy draws in the
    same order (3 scales U[1-s, 1/(1-s)], 6 shears, 3 translations, 3 integer angles), same fp32 products
    Rx @ Ry @ Rz @ S.  Axis convention of the reference: arguments in [z, y, x] order, matrix rows in (x, y, z)."""
    scale, translate, rotate, shear = _triple(scale), _triple(translate), _triple(rotate), _triple(shear)
    diag = [np.random.uniform(low=1 - s, high=1 / (1 - s)) for s in scale]
    off = [np.random.uniform(-shear[i // 2], shear[i // 2]) for i in range(6)]     # xy, xz, yx, yz, zx, zy
    tr = [np.random.uniform(-t, t) for t in translate]
    S = torch.tensor([[diag[0], off[0], off[1], tr[0]],
                      [off[2], diag[1], off[3], tr[1]],
                      [off[4], off[5], diag[2], tr[2]],
                      [0, 0, 0, 1]]).float()
    ang = [(float(np.random.randint(-r, max(r, 1))) / 180.) * math.pi for r in rotate]
    mats = []
    for axis, a in enumerate(ang):
        c, s = math.cos(a), math.sin(a)
        i, j = [(1, 2), (0, 2), (0, 1)][axis]          # plane the rotation acts in: about x -> (y,z); y -> (x,z); z -> (x,y)
        R = [[1.0 if r == q else 0.0 for q in range(4)] for r in range(4)]
        R[i][i], R[i][j], R[j][i], R[j][j] = c, -s, s, c
        mats.append(torch.tensor(R).float())
    theta = torch.mm(torch.mm(torch.mm(mats[0], mats[1]), mats[2]), S)
    return theta[0:3, :].contiguous()


def draw_affine_theta_2d(scale=0.3, rotate=180, translate=0):
    """The random 2x3 matrix of ``random_scale_rotate_translate_2d`` (augmentation.py:192-214): six np.random.random()
    draws (x/y scale, x/y shear, x/y translation), then one integer angle; fp32 product S @ R."""
    scale = [scale] * 2 if isinstance(scale, (int, float)) else list(scale)
    translate = [translate] * 2 if isinstance(translate, (int, float)) else list(translate)
    sx = 1 - scale[0] + np.random.random() * 2 * scale[0]
    sy = 1 - scale[1] + np.random.random() * 2 * scale[1]
    hx = np.random.random() * 2 * scale[0] - scale[0]
    hy = np.random.random() * 2 * scale[1] - scale[1]
    tx = np.random.random() * 2 * translate[0] - translate[0]
    ty = np.random.random() * 2 * translate[1] - translate[1]
    S = torch.tensor([[sx, hx, tx], [hy, sy, ty], [0, 0, 1]]).float()
    a = (float(np.random.randint(-rotate, max(rotate, 1))) / 180.) * math.pi
    R = torch.tensor([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]]).float()
    return torch.mm(S, R)[0:2, :].contiguous()


def embed_theta_2d(theta):
    """A 2x3 theta as the 3x4 of the volume gather on a D = 1 grid: the z tap weight is exactly 0, so trilinear
    sampling of the one plane is bilinear sampling."""
    t = torch.as_tensor(theta, dtype=torch.float32).reshape(2, 3)
    out = torch.zeros(3, 4)
    out[:2, :2], out[:2, 3], out[2, 2] = t[:, :2], t[:, 2], 1.0
    return out


def _as_volume(t):
    """[1, C, H, W] -> the [1, C, 1, H, W] view the volume kernels take."""
    return None if t is None else t.unsqueeze(2)


def random_scale_rotate_translate_2d(tensor_img, tensor_lab, scale, rotate, translate):
    """augmentation.py:192-223 on the whole slice."""
    theta = embed_theta_2d(draw_affine_theta_2d(scale, rotate, translate))
    size = [1] + list(tensor_img.shape[2:])
    img, lab, _ = resample(_as_volume(tensor_img), _as_volume(tensor_lab), (0, 0, 0), size, theta, (0, 0, 0), size)
    return img.squeeze(2), lab.squeeze(2)


def crop_2d(tensor_img, tensor_lab, crop_size, mode):
    """augmentation.py:297-317 (slicing clamps at the slice border, as Python slices do)."""
    assert mode in ['random', 'center'], "Invalid Mode, should be 'random' or 'center'"
    crop_size = [crop_size] * 2 if isinstance(crop_size, int) else list(crop_size)
    shape = list(tensor_img.shape[2:])
    if mode == 'random':
        org = _crop_origin_random(shape, crop_size)
    else:
        org = [(s - c) // 2 for s, c in zip(shape, crop_size)]
    if min(org) < 0:
        raise ValueError("centre crop larger than the slice (the reference's negative slice start is not supported)")
    size = [min(c, s - o) for c, s, o in zip(crop_size, shape, org)]
    lab = _lab(tensor_lab)
    img, olab, _ = resample(_as_volume(tensor_img), _as_volume(lab), [0] + org, [1] + size, None, (0, 0, 0), [1] + size,
                            out_label_dtype=lab.dtype)
    return img.squeeze(2), olab.squeeze(2)


def random_scale_rotate_translate_3d(tensor_img, tensor_lab, scale=0.3, rotate=45, translate=0.1, shear=0.05):
    """augmentation.py:226-291 on the whole input volume."""
    _vol(tensor_img, tensor_lab)
    theta = draw_affine_theta(scale, rotate, translate, shear)
    size = list(tensor_img.shape[2:])
    img, lab, _ = resample(tensor_img, tensor_lab, (0, 0, 0), size, theta, (0, 0, 0), size)
    return img, lab


def _crop_origin_random(shape, crop_size):
    diffs = [s - c for s, c in zip(shape, crop_size)]
    return [int(np.random.randint(0, max(d, 1))) for d in diffs]      # z, y, x — the reference's draw order


def crop_3d(tensor_img, tensor_lab, crop_size, mode):
    """augmentation.py:320-343 (slicing clamps at the volume border, as Python slices do)."""
    assert mode in ['random', 'center'], "Invalid Mode, should be 'random' or 'center'"
    _vol(tensor_img, tensor_lab)
    crop_size = _triple(crop_size) if isinstance(crop_size, int) else list(crop_size)
    shape = list(tensor_img.shape[2:])
    if mode == 'random':
        org = _crop_origin_random(shape, crop_size)
    else:
        org = [(s - c) // 2 for s, c in zip(shape, crop_size)]
    if min(org) < 0:
        raise ValueError("centre crop larger than the volume (the reference's negative slice start is not supported)")
    size = [min(c, s - o) for c, s, o in zip(crop_size, shape, org)]
    img, lab, _ = resample(tensor_img, tensor_lab, org, size, None, (0, 0, 0), size)
    return img, lab


def crop_around_coordinate_3d(tensor_img, tensor_lab, crop_size, coordinate, mode):
    """augmentation.py:346-383."""
    assert mode in ['random', 'center'], "Invalid Mode, should be 'random' or 'center'"
    _vol(tensor_img, tensor_lab)
    crop_size = _triple(crop_size) if isinstance(crop_size, int) else list(crop_size)
    shape = list(tensor_img.shape[2:])
    org = []
    for c, s, k in zip(coordinate, shape, crop_size):
        if mode == 'random':
            lo, hi = max(0, c - k), min(s - k, c + k)
            org.append(int(np.random.randint(lo, hi)))
        else:
            org.append(min(max(0, c - math.ceil(k / 2)), s - k))
    size = [min(c, s - o) for c, s, o in zip(crop_size, shape, org)]
    img, lab, _ = resample(tensor_img, tensor_lab, org, size, None, (0, 0, 0), size)
    return img, lab


def mirror(tensor_img, axis=0):
    """torch.flip(dims=[2+axis]) (augmentation.py:176-197) for an image or a label map, volume or slice."""
    if tensor_img.dim() == 4:
        assert axis in [0, 1], "axis should be either 0 or 1 for 2D images"
        return mirror(_as_volume(tensor_img), axis + 1).squeeze(2)
    assert axis in [0, 1, 2], "axis should be either 0, 1 or 2 for volume images"
    _vol(tensor_img)
    flips = [axis == 0, axis == 1, axis == 2]
    size = list(tensor_img.shape[2:])
    if tensor_img.dtype == torch.float32:
        return resample(tensor_img, None, (0, 0, 0), size, None, (0, 0, 0), size, flips)[0]
    lab = _lab(tensor_img)      # label map: the label slot of the gather alone
    return resample(None, lab, (0, 0, 0), size, None, (0, 0, 0), size, flips, out_label_dtype=lab.dtype)[1]


# ----------------------------------------------------------------------------- intensity
def gaussian_noise(tensor_img, std, mean=0):
    """augmentation.py:14-16.  The reference draws the noise volume on the host and copies it; here the normals come from
    a counter-based Philox generator in the kernel, keyed by one integer drawn from torch's CPU generator."""
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    return _pointwise(tensor_img, OP_NOISE, a=[std], b=[mean], rows=1, seed=seed)[0]


def gaussian_kernel_1d(kernel_size, sigma):
    """1-D factor of generate_3d_gaussian_kernel / generate_2d_gaussian_kernel (augmentation.py:18-44): the normalised
    dense kernel is its outer cube / outer square."""
    r = torch.arange(-kernel_size // 2 + 1, kernel_size // 2 + 1, dtype=torch.float32)
    w = torch.exp(-(r ** 2) / (2 * float(sigma) ** 2))
    return (w / w.sum()).contiguous()


def _blur(tensor_img, sigma, want_stats=False, per_channel=False):
    x = _img(tensor_img)
    kernel_size = 2 * math.ceil(3 * sigma) + 1
    w = gaussian_kernel_1d(kernel_size, sigma)
    y = torch.empty_like(x)
    rows = _rows(x.shape[1], per_channel)
    so = new_stats(rows, x.device) if want_stats else None
    if x.dim() == 4:
        _, C, H, W = x.shape
        call("b200seg_aug_gaussian_blur2d", x.data_ptr(), y.data_ptr(), C, H, W, w.data_ptr(), kernel_size,
             None if so is None else so.data_ptr(), rows, _stream())
        return y, so
    _, C, D, H, W = x.shape
    call("b200seg_aug_gaussian_blur", x.data_ptr(), y.data_ptr(), C, D, H, W, w.data_ptr(), kernel_size,
         None if so is None else so.data_ptr(), rows, _stream())
    return y, so


def gaussian_blur(tensor_img, sigma_range=[0.5, 1.0]):
    """augmentation.py:46-64."""
    sigma = float(torch.rand(1) * (sigma_range[1] - sigma_range[0]) + sigma_range[0])
    return _blur(tensor_img, sigma)[0]


def brightness_additive(tensor_img, std, mean=0, per_channel=False):
    """augmentation.py:66-85."""
    C = tensor_img.shape[1] if per_channel else 1
    r = torch.normal(mean, std, size=(1, C) + (1,) * (tensor_img.dim() - 2))
    return _pointwise(tensor_img, OP_ADD, a=r, rows=C)[0]


def brightness_multiply(tensor_img, multiply_range=[0.7, 1.3], per_channel=False):
    """augmentation.py:88-101."""
    assert multiply_range[1] > multiply_range[0], 'Invalid range'
    C = tensor_img.shape[1] if per_channel else 1
    r = torch.rand(size=(1, C) + (1,) * (tensor_img.dim() - 2)) * (multiply_range[1] - multiply_range[0]) + multiply_range[0]
    return _pointwise(tensor_img, OP_MUL, a=r, rows=C)[0]


def _check_rows(C, per_channel):
    if C > 1 and not per_channel:
        # the reference broadcasts a [C,1] random vector against a [1,N] view and then fails to reshape
        raise ValueError("multi-channel images need per_channel=True (the reference's own view() fails otherwise)")
    return C


def _gamma(tensor_img, g, rows, stats=None, retain_stats=True, want_stats=False):
    if stats is None:
        stats = image_stats(tensor_img, per_channel=rows > 1)
    y, s1 = _pointwise(tensor_img, OP_GAMMA_POW, a=g, rows=rows, stats_in=stats, want_stats=retain_stats or want_stats)
    if retain_stats:
        y, s1 = _pointwise(y, OP_RENORM, rows=rows, stats_in=s1, stats_in2=stats, want_stats=want_stats)
    return y, s1


def gamma(tensor_img, gamma_range=(0.5, 2), per_channel=False, retain_stats=True):
    """augmentation.py:104-137."""
    C = _check_rows(tensor_img.shape[1], per_channel)
    g = torch.rand(C, 1) * (gamma_range[1] - gamma_range[0]) + gamma_range[0]
    return _gamma(tensor_img, g, C, retain_stats=retain_stats)[0]


def _contrast(tensor_img, f, rows, stats=None, preserve_range=True, want_stats=False):
    if stats is None:
        stats = image_stats(tensor_img, per_channel=rows > 1)
    return _pointwise(tensor_img, OP_CONTRAST, a=f, b=[1.0 if preserve_range else 0.0] * rows, rows=rows, stats_in=stats,
                      want_stats=want_stats)


def contrast(tensor_img, contrast_range=(0.65, 1.5), per_channel=False, preserve_range=True):
    """augmentation.py:139-173."""
    C = _check_rows(tensor_img.shape[1], per_channel)
    f = torch.rand(C, 1) * (contrast_range[1] - contrast_range[0]) + contrast_range[0]
    return _contrast(tensor_img, f, C, preserve_range=preserve_range)[0]


# ----------------------------------------------------------------------------- the training branch as one plan
class TrainAugment3D:
    """The ``mode == 'train'`` branch of the 3D datasets' ``__getitem__`` (dataset_kits.py:116-153; the other 3D
    datasets use the same sequence): crop trick + affine (p=0.2) or random crop, brightness / gamma / contrast (p=0.2
    each), mirrors about W, H, D (p=0.3 each), blur (p=0.2), noise (p=0.2).

    ``plan()`` consumes ``np.random`` / ``torch`` CPU random numbers exactly as the reference does (same calls, same
    order), ``apply()`` executes a plan on the device.  Mirrors are folded into the gather: the intensity ops between
    the geometry and the flips are voxelwise with whole-image statistics, the blur kernel is symmetric, so moving the
    flips forward changes nothing but floating-point summation order."""

    def __init__(self, training_size, scale=0.3, rotate=45, translate=0.1, shear=0.05, margin=60):
        self.size = list(training_size)
        self.scale, self.rotate, self.translate, self.shear, self.margin = scale, rotate, translate, shear, margin

    def plan(self, volume_shape, channels=1):
        shape = list(volume_shape)
        p = {}
        if np.random.random() < 0.2:
            big = [s + self.margin for s in self.size]
            org = _crop_origin_random(shape, big)
            sub = [min(b, s - o) for b, s, o in zip(big, shape, org)]
            p["sub_origin"], p["sub_size"] = org, sub
            p["theta"] = draw_affine_theta(self.scale, self.rotate, self.translate, self.shear)
            p["out_origin"] = [(s - c) // 2 for s, c in zip(sub, self.size)]
        else:
            org = _crop_origin_random(shape, self.size)
            p["sub_origin"], p["sub_size"], p["theta"], p["out_origin"] = org, list(self.size), None, [0, 0, 0]
        if min(p["out_origin"]) < 0 or any(o + c > s for o, c, s in zip(p["out_origin"], self.size, p["sub_size"])):
            raise ValueError("volume %s is smaller than the training size %s" % (shape, self.size))
        C = channels
        p["brightness"] = (torch.rand(size=(1, 1, 1, 1, 1)) * 0.6 + 0.7) if np.random.random() < 0.2 else None
        p["gamma"] = (torch.rand(C, 1) * (1.5 - 0.7) + 0.7) if np.random.random() < 0.2 else None
        p["contrast"] = (torch.rand(C, 1) * (1.5 - 0.65) + 0.65) if np.random.random() < 0.2 else None
        fw = np.random.random() < 0.3      # axis=2
        fh = np.random.random() < 0.3      # axis=1
        fd = np.random.random() < 0.3      # axis=0
        p["flips"] = (fd, fh, fw)
        p["blur_sigma"] = float(torch.rand(1) * 0.5 + 0.5) if np.random.random() < 0.2 else None
        if np.random.random() < 0.2:
            p["noise_std"] = np.random.random() * 0.1
            p["noise_seed"] = int(torch.randint(0, 2 ** 62, (1,)).item())
        else:
            p["noise_std"] = None
        return p

    def apply(self, tensor_img, tensor_lab, p):
        _vol(tensor_img, tensor_lab)
        C = tensor_img.shape[1]
        need_stats = p["gamma"] is not None or p["contrast"] is not None
        img, lab, st = resample(tensor_img, tensor_lab, p["sub_origin"], p["sub_size"], p["theta"], p["out_origin"],
                                self.size, p["flips"], want_stats=need_stats and p["brightness"] is None)
        if p["brightness"] is not None:
            img, st = _pointwise(img, OP_MUL, a=p["brightness"], rows=1, want_stats=need_stats)
        if p["gamma"] is not None:
            _check_rows(C, False)
            img, st = _gamma(img, p["gamma"], 1, stats=st, want_stats=p["contrast"] is not None)
        if p["contrast"] is not None:
            _check_rows(C, False)
            img, _ = _contrast(img, p["contrast"], 1, stats=st)
        if p["blur_sigma"] is not None:
            img, _ = _blur(img, p["blur_sigma"])
        if p["noise_std"] is not None:
            img, _ = _pointwise(img, OP_NOISE, a=[p["noise_std"]], b=[0.0], rows=1, seed=p["noise_seed"])
        return img, lab

    def __call__(self, tensor_img, tensor_lab):
        _vol(tensor_img, tensor_lab)                      # before any draw
        if not tensor_img.is_cuda:
            raise B200SegError("b200seg.augmentation runs on an H100 only — there is no CPU fallback")
        return self.apply(tensor_img, tensor_lab, self.plan(tensor_img.shape[2:], tensor_img.shape[1]))


# ----------------------------------------------------------------------------- the 2D slice branch for a whole batch
_ROW = struct.Struct("<QQQiiQfff6fiii")          # b200seg_aug2d_row (include/b200seg.h), 88 bytes
assert _ROW.size == 88


class TrainAugment2D:
    """The ``mode == 'train'`` branch of the 2D ACDC dataset's ``__getitem__`` (dataset_acdc.py:128-142), for a batch
    of B slices of their own H x W: gaussian_noise -> brightness_additive -> gamma(retain_stats) ->
    random_scale_rotate_translate_2d -> crop_2d(random), every op applied (no coin flips in that branch).

    ``plan()`` makes one slice's draws in the order of the public functions above (noise key, brightness, gamma, the six
    affine numbers and the angle, the two crop offsets).  The numpy draws, and so the geometry and the crop, are the
    reference's for the same ``np.random`` state.  The torch draws are not: the reference's ``torch.randn`` of the
    whole slice consumes as many numbers as the slice has pixels, where the noise here is a counter-based Philox
    stream keyed by one ``torch.randint`` draw (the key :func:`gaussian_noise` uses).

    ``apply()`` runs the plans as one batch in three launches (``b200seg_aug2d_train``): two per-slice statistics
    passes and one gather of the h x w crops.  It returns ``img [B, 1, h, w]`` fp32 and ``lab [B, 1, h, w]`` int64,
    the layout ``UNet2D`` and ``DiceCELoss`` take.  The slice statistics never leave the device, and a given plan gives
    the same bits on every run."""

    def __init__(self, training_size, scale=0.3, rotate=180, translate=0, gaussian_noise_std=0.02,
                 additive_brightness_std=0.7, gamma_range=(0.5, 1.6)):
        self.size = [training_size] * 2 if isinstance(training_size, int) else list(training_size)
        self.scale, self.rotate, self.translate = scale, rotate, translate
        self.noise_std, self.brightness_std, self.gamma_range = float(gaussian_noise_std), additive_brightness_std, gamma_range

    def plan(self, slice_shape):
        H, W = [int(s) for s in slice_shape[-2:]]
        h, w = self.size
        if H < h or W < w:
            raise ValueError("slice %dx%d is smaller than the training size %dx%d" % (H, W, h, w))
        p = {"noise_std": self.noise_std}
        p["noise_key"] = int(torch.randint(0, 2 ** 62, (1,)).item())
        p["beta"] = float(torch.normal(0, self.brightness_std, size=(1, 1, 1, 1)))
        p["gamma"] = float(torch.rand(1, 1) * (self.gamma_range[1] - self.gamma_range[0]) + self.gamma_range[0])
        p["theta"] = draw_affine_theta_2d(self.scale, self.rotate, self.translate)
        p["crop"] = _crop_origin_random([H, W], self.size)
        return p

    @staticmethod
    def _slice(t, what):
        _need_cuda(t)
        if t.dim() == 4:
            if t.shape[0] != 1 or t.shape[1] != 1:
                raise ValueError("%s must be [H, W] or [1, 1, H, W] (one channel), got %s" % (what, list(t.shape)))
            t = t[0, 0]
        elif t.dim() != 2:
            raise ValueError("%s must be [H, W] or [1, 1, H, W], got %s" % (what, list(t.shape)))
        return t.contiguous()

    def apply(self, images, labels, plans, y1_out=None):
        """y1_out (optional, for tests): a list of contiguous fp32 [H, W] tensors on the images' device, one per slice,
        that receive each slice's noisy, brightened image y1 = x + std * n + beta."""
        return self._prepare(images, labels, plans, y1_out)()

    def _prepare(self, images, labels, plans, y1_out=None):
        """Check the inputs, pack and upload the table, allocate the outputs; returns a function that launches the
        batch (``b200seg_aug2d_train``) and returns (img, lab)."""
        if not (len(images) == len(labels) == len(plans)) or not images:
            raise ValueError("images, labels and plans must be non-empty lists of the same length")
        imgs = [self._slice(t, "image") for t in images]
        labs = [self._slice(t, "label map") for t in labels]
        for x, l in zip(imgs, labs):
            if x.dtype != torch.float32:
                raise TypeError("images are fp32 (the reference augments before autocast), got %s" % x.dtype)
            if x.shape != l.shape:
                raise ValueError("image %s and label map %s differ in shape" % (list(x.shape), list(l.shape)))
            if x.shape[0] < self.size[0] or x.shape[1] < self.size[1]:
                raise ValueError("slice %s is smaller than the training size %s" % (list(x.shape), self.size))
        if y1_out is not None:
            if len(y1_out) != len(imgs):
                raise ValueError("y1_out needs one tensor per slice")
            for x, y in zip(imgs, y1_out):
                _need_cuda(y)
                if y.device != x.device or y.dtype != torch.float32 or y.shape != x.shape or not y.is_contiguous():
                    raise ValueError("y1_out tensors are contiguous fp32 [H, W] on the images' device, one per slice; got "
                                     "%s %s %s for a %s slice" % (y.dtype, list(y.shape), y.device, list(x.shape)))
        lab_dt = torch.uint8 if all(l.dtype == torch.uint8 for l in labs) else torch.int64
        labs = [l.to(lab_dt) for l in labs]
        h, w = self.size
        B, dev = len(imgs), imgs[0].device
        table = bytearray()
        for i, (x, l, p) in enumerate(zip(imgs, labs, plans)):
            oy, ox = p["crop"]
            if not (0 <= oy <= x.shape[0] - h and 0 <= ox <= x.shape[1] - w):
                raise ValueError("crop origin %s outside slice %s" % ((oy, ox), list(x.shape)))
            y1 = 0 if y1_out is None else y1_out[i].data_ptr()
            th = torch.as_tensor(p["theta"], dtype=torch.float32).reshape(6).tolist()
            table += _ROW.pack(x.data_ptr(), l.data_ptr(), y1, x.shape[0], x.shape[1], p["noise_key"] & 0xFFFFFFFFFFFFFFFF,
                               p["noise_std"], p["beta"], p["gamma"], *th, oy, ox, 0)
        rows = torch.frombuffer(table, dtype=torch.uint8)
        if dev.type == "cuda":
            rows = rows.pin_memory()
        rows = rows.to(dev, non_blocking=True)          # the one host-to-device copy of the call
        max_elems = max(x.numel() for x in imgs)
        ws_bytes = int(load_lib().b200seg_aug2d_workspace(B, max_elems))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        out_img = torch.empty(B, 1, h, w, dtype=torch.float32, device=dev)
        out_lab = torch.empty(B, 1, h, w, dtype=torch.int64, device=dev)

        def launch():
            call("b200seg_aug2d_train", rows.data_ptr(), B, max_elems, labs[0].element_size(), h, w, out_img.data_ptr(),
                 out_lab.data_ptr(), ws.data_ptr(), ws_bytes, _stream())
            return out_img, out_lab
        launch.inputs = imgs          # the (possibly copied) slices the table points at live as long as the launcher
        return launch

    def __call__(self, images, labels):
        imgs = [self._slice(t, "image") for t in images]       # shapes and devices are checked before any draw
        return self.apply(imgs, labels, [self.plan(t.shape) for t in imgs])

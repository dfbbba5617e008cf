"""CPU: the 2D augmentation oracle against the fixtures the unmodified reference produced (tests/golden/augment2d_*.pt),
the random draws of TrainAugment2D.plan(), its input checks, and its launch count — no kernel runs here."""
import os

import numpy as np
import pytest
import torch

import b200seg
from b200seg import augmentation as aug
from oracle import augmentation2d as o2

CFG = dict(scale=0.3, rotate=180, translate=0, gaussian_noise_std=0.02, additive_brightness_std=0.7, gamma_range=[0.5, 1.6])


@pytest.fixture(scope="module")
def ops_fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "augment2d_ops.pt"), weights_only=False)


@pytest.fixture(scope="module")
def train_fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "augment2d_train.pt"), weights_only=False)


def _md(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def test_plan_draws_in_documented_order():
    """Per slice, in batch order: torch randint key, torch normal, torch rand, six np.random.random() + one randint,
    two crop randints."""
    ta = aug.TrainAugment2D([256, 256], **CFG)
    shapes = [(266, 300), (420, 480), (300, 266)]
    np.random.seed(5)
    torch.manual_seed(5)
    plans = [ta.plan(s) for s in shapes]
    np.random.seed(5)
    torch.manual_seed(5)
    for (H, W), p in zip(shapes, plans):
        assert p["noise_key"] == int(torch.randint(0, 2 ** 62, (1,)).item())
        assert p["beta"] == float(torch.normal(0, 0.7, size=(1, 1, 1, 1)))
        assert p["gamma"] == float(torch.rand(1, 1) * (1.6 - 0.5) + 0.5)
        r6, ang = o2.draws_affine_2d(0.3, 180, 0)
        assert np.array_equal(p["theta"].numpy(), o2.theta_from_draws(r6, ang))
        assert p["crop"] == [int(np.random.randint(0, max(H - 256, 1))), int(np.random.randint(0, max(W - 256, 1)))]
        assert p["noise_std"] == np.float32(0.02)


def test_plan_geometry_is_the_references(train_fx):
    """The numpy stream alone fixes theta and the crop: the same np.random seed gives the matrix and the crop origin
    the reference's own functions used."""
    c = train_fx["cfg"]
    ta = aug.TrainAugment2D(c["training_size"], c["scale"], c["rotate"], c["translate"], c["gaussian_noise_std"],
                            c["additive_brightness_std"], c["gamma_range"])
    for case in train_fx["cases"]:
        np.random.seed(case["seed"])
        p = ta.plan(case["img_in"].shape)
        assert np.array_equal(p["theta"].numpy(), case["theta"].numpy()), case["seed"]
        assert p["crop"] == case["crop_origin"], case["seed"]


def test_oracle_ops_match_reference(ops_fx):
    for c in ops_fx["slices"]:
        img, lab = c["img"][None].numpy(), c["lab"].numpy()
        for a in c["affine"]:
            theta = o2.theta_from_draws(*a["draws"])
            assert np.array_equal(theta, a["theta"].numpy())
            oi, ol = o2.scale_rotate_translate_2d(img, lab, theta)
            assert _md(oi[0], a["img"]) < 5e-5 and (ol != a["lab"].numpy()).mean() < 2e-3
        oi, ol = o2.crop_2d(img, lab, c["crop_origin"], ops_fx["crop"])
        assert _md(oi[0], c["crop_img"]) == 0 and np.array_equal(ol, c["crop_lab"].numpy())
        assert _md(img[0] + c["brightness_additive"]["param"], c["brightness_additive"]["out"]) < 2e-5
        assert _md(img[0] * c["brightness_multiply"]["param"], c["brightness_multiply"]["out"]) < 2e-5
        assert _md(o2.gamma(img, c["gamma"]["param"])[0], c["gamma"]["out"]) < 2e-5
        assert _md(o2.gamma(img, c["gamma_no_retain"]["param"], retain_stats=False)[0], c["gamma_no_retain"]["out"]) < 2e-5
        assert _md(o2.contrast(img, c["contrast"]["param"])[0], c["contrast"]["out"]) < 2e-5
        assert _md(o2.gaussian_blur(img, c["blur"]["param"])[0], c["blur"]["out"]) < 2e-5


def test_oracle_branch_matches_reference(train_fx):
    size = train_fx["cfg"]["training_size"]
    for case in train_fx["cases"]:
        oi, ol = o2.train_branch(case["img_in"].numpy(), case["lab_in"].numpy(), case["beta"], case["gamma"],
                                 case["theta"].numpy(), case["crop_origin"], size)
        assert _md(oi, case["img"]) < 5e-5, case["seed"]
        assert (ol != case["lab"].numpy()).mean() < 2e-3, case["seed"]


def test_rejections(monkeypatch):
    ta = aug.TrainAugment2D([64, 64], **CFG)
    x, l = torch.zeros(80, 90), torch.zeros(80, 90, dtype=torch.uint8)
    with pytest.raises(b200seg.B200SegError):            # CPU tensors: there is no CPU path
        ta([x], [l])
    with pytest.raises(b200seg.B200SegError):
        aug.gaussian_noise(x[None, None], std=0.1)
    monkeypatch.setattr(aug, "_need_cuda", lambda t: None)
    with pytest.raises(ValueError):                      # C != 1
        ta([torch.zeros(1, 3, 80, 90)], [torch.zeros(1, 1, 80, 90, dtype=torch.uint8)])
    with pytest.raises(ValueError):                      # smaller than the crop (the reference would return a short crop)
        ta([torch.zeros(80, 60)], [torch.zeros(80, 60, dtype=torch.uint8)])
    with pytest.raises(ValueError):
        ta.plan((63, 200))
    with pytest.raises(ValueError):                      # image and label map of different shapes
        ta.apply([x], [torch.zeros(80, 91, dtype=torch.uint8)], [ta.plan((80, 90))])


def test_abi_calls_do_not_grow_with_batch(monkeypatch):
    """One batch is one host-to-device table copy and one C-ABI call (three launches), whatever B."""
    monkeypatch.setattr(aug, "_need_cuda", lambda t: None)
    monkeypatch.setattr(aug, "_stream", lambda: 0)
    ta = aug.TrainAugment2D([32, 32], **CFG)
    counts = {}
    for B in (1, 8, 32):
        calls = []
        monkeypatch.setattr(aug, "call", lambda name, *a: calls.append(name))
        g = torch.Generator().manual_seed(B)
        imgs = [torch.randn(40 + i % 7, 36 + i % 5, generator=g) for i in range(B)]
        labs = [torch.zeros(t.shape, dtype=torch.uint8) for t in imgs]
        out_i, out_l = ta(imgs, labs)
        assert out_i.shape == (B, 1, 32, 32) and out_l.shape == (B, 1, 32, 32) and out_l.dtype == torch.int64
        counts[B] = list(calls)
    assert counts[1] == counts[8] == counts[32] == ["b200seg_aug2d_train"]
    assert b200seg._lib._KERNELS["b200seg_aug2d_train"] == 3


def test_volume_functions_reject_slices_before_any_call(monkeypatch):
    """A [1, C, H, W] tensor never reaches the volume gather (it reads three-entry geometry arrays), and is rejected
    before any random draw."""
    monkeypatch.setattr(aug, "_need_cuda", lambda t: None)
    monkeypatch.setattr(aug, "_stream", lambda: 0)
    calls = []
    monkeypatch.setattr(aug, "call", lambda name, *a: calls.append(name))
    img, lab = torch.zeros(1, 1, 70, 90), torch.zeros(1, 1, 70, 90, dtype=torch.uint8)
    np.random.seed(0)
    state = np.random.get_state()[1].copy()
    cases = [lambda: aug.random_scale_rotate_translate_3d(img, lab),
             lambda: aug.crop_3d(img, lab, [48, 48, 48], "random"),
             lambda: aug.crop_3d(img, lab, [48, 48, 48], "center"),
             lambda: aug.crop_around_coordinate_3d(img, lab, [8, 8, 8], (30, 30, 30), "random"),
             lambda: aug.resample(img, lab, (0, 0, 0), [1, 70, 90], None, (0, 0, 0), [1, 70, 90]),
             lambda: aug.resample(img[:, :, None], lab[:, :, None], (0, 0), [70, 90], None, (0, 0), [70, 90]),
             lambda: aug.TrainAugment3D([48, 48, 48])(img, lab),
             lambda: aug.TrainAugment3D([48, 48, 48]).apply(img, lab, {})]
    for k, fn in enumerate(cases):
        with pytest.raises(ValueError):
            fn()
        assert calls == [], k
    assert np.array_equal(np.random.get_state()[1], state)
    # the 2D functions still reach the gather, through their [1, C, 1, H, W] views
    aug.crop_2d(img, lab, [48, 48], "center")
    aug.mirror(img, 1)
    assert calls == ["b200seg_aug_resample"] * 2


def test_y1_out_is_checked(monkeypatch):
    monkeypatch.setattr(aug, "_need_cuda", lambda t: None)
    monkeypatch.setattr(aug, "_stream", lambda: 0)
    calls = []
    monkeypatch.setattr(aug, "call", lambda name, *a: calls.append(name))
    ta = aug.TrainAugment2D([32, 32], **CFG)
    x, l = torch.zeros(40, 36), torch.zeros(40, 36, dtype=torch.uint8)
    plans = [ta.plan(x.shape)]
    for bad in ([torch.zeros(40, 35)], [torch.zeros(40, 36, dtype=torch.float64)], [torch.zeros(36, 40).t()], []):
        with pytest.raises(ValueError):
            ta.apply([x], [l], plans, y1_out=bad)
    assert calls == []
    ta.apply([x], [l], plans, y1_out=[torch.zeros(40, 36)])
    assert calls == ["b200seg_aug2d_train"]

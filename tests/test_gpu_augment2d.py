"""GPU: the 2D augmentation functions and the batched slice branch (b200seg_aug2d_train) against the fixtures the
unmodified reference produced (tests/golden/augment2d_*.pt), the float64 oracle at the ACDC batch shape, and the chain
of public 2D functions."""
import os

import numpy as np
import pytest
import torch

import b200seg
from b200seg import augmentation as aug
from oracle import augmentation2d as o2

pytestmark = pytest.mark.gpu
TOL = 5e-5          # the bars of the 3D augmentation tests: images, and the share of label pixels that may differ
LAB_TOL = 2e-3
ACDC = dict(scale=0.3, rotate=180, translate=0, gaussian_noise_std=0.02, additive_brightness_std=0.7, gamma_range=[0.5, 1.6])


@pytest.fixture(scope="module")
def ops_fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "augment2d_ops.pt"), weights_only=False)


@pytest.fixture(scope="module")
def train_fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "augment2d_train.pt"), weights_only=False)


def _md(a, b):
    return float((torch.as_tensor(np.asarray(a.detach().cpu() if torch.is_tensor(a) else a)).double()
                  - torch.as_tensor(np.asarray(b)).double()).abs().max())


def _mis(a, b):
    return float((a.cpu().long() != torch.as_tensor(np.asarray(b)).long()).float().mean())


def _ragged(B, seed, h_range=(266, 420), w_range=(266, 480)):
    rng = np.random.RandomState(seed)
    out = []
    for i in range(B):
        H, W = int(rng.randint(*h_range)), int(rng.randint(*w_range))
        img, lab = o2.make_slice(H, W, 4, seed=seed * 100 + i)
        out.append((img.cuda(), lab.cuda()))
    return [i for i, _ in out], [l for _, l in out]


def test_functions_match_reference_fixture(ops_fx):
    for k, c in enumerate(ops_fx["slices"]):
        img, lab = c["img"][None, None].cuda(), c["lab"][None, None].cuda()
        for a in c["affine"]:
            np.random.seed(a["seed"])
            oi, ol = aug.random_scale_rotate_translate_2d(img, lab, *a["args"])
            assert oi.shape == img.shape and ol.dtype == torch.int64
            assert _md(oi[0, 0], a["img"]) < TOL and _mis(ol[0, 0], a["lab"]) < LAB_TOL, a["seed"]
        np.random.seed(c["crop_seed"])
        ci, cl = aug.crop_2d(img, lab, ops_fx["crop"], mode="random")
        assert torch.equal(ci[0, 0].cpu(), c["crop_img"]) and torch.equal(cl[0, 0].cpu(), c["crop_lab"])
        oy, ox = [(s - k) // 2 for s, k in zip(img.shape[2:], ops_fx["crop"])]
        ci, _ = aug.crop_2d(img, lab, ops_fx["crop"], mode="center")
        assert torch.equal(ci, img[:, :, oy:oy + 48, ox:ox + 48])
        # the public functions draw their parameter as the reference did (the fixture ran them in this order)
        torch.manual_seed(60 + k)
        outs = {"brightness_additive": aug.brightness_additive(img, std=0.7),
                "brightness_multiply": aug.brightness_multiply(img, multiply_range=[0.7, 1.3]),
                "gamma": aug.gamma(img, gamma_range=[0.5, 1.6], retain_stats=True),
                "gamma_no_retain": aug.gamma(img, gamma_range=[0.5, 1.6], retain_stats=False),
                "contrast": aug.contrast(img, contrast_range=[0.65, 1.5]),
                "blur": aug.gaussian_blur(img, sigma_range=[0.5, 1.0])}
        for name, y in outs.items():
            assert y.shape == img.shape and _md(y[0, 0], c[name]["out"]) < TOL, name
        for ax in (0, 1):
            assert torch.equal(aug.mirror(img, ax), torch.flip(img, [2 + ax]))
            assert torch.equal(aug.mirror(lab, ax), torch.flip(lab, [2 + ax]))


def test_branch_matches_reference_fixture(train_fx):
    c = train_fx["cfg"]
    ta = aug.TrainAugment2D(c["training_size"], c["scale"], c["rotate"], c["translate"], c["gaussian_noise_std"],
                            c["additive_brightness_std"], c["gamma_range"])
    imgs, labs, plans = [], [], []
    for case in train_fx["cases"]:
        np.random.seed(case["seed"])
        p = ta.plan(case["img_in"].shape)
        # the torch draws differ from the reference's (its noise consumes H*W normals): use the ones it drew
        p["beta"], p["gamma"] = case["beta"], case["gamma"]
        imgs.append(case["img_in"].cuda())
        labs.append(case["lab_in"].cuda())
        plans.append(p)
    oi, ol = ta.apply(imgs, labs, plans)
    for b, case in enumerate(train_fx["cases"]):
        assert _md(oi[b, 0], case["img"]) < TOL, case["seed"]
        assert _mis(ol[b, 0], case["lab"]) < LAB_TOL, case["seed"]


def test_acdc_batch_matches_fp64_oracle():
    """B = 32 ragged slices of 266-420 x 266-480 at the ACDC settings, slice by slice against the float64 oracle fed
    the image plus the noise the same key gives through gaussian_noise.  At these extents a float32 sampling position
    is only defined to ~1e-4 px (the reference's own positions are float32), so each pixel may also differ by what a
    2-ulp move of its position changes in the oracle."""
    imgs, labs = _ragged(32, seed=1)
    ta = aug.TrainAugment2D([256, 256], **ACDC)
    np.random.seed(2)
    torch.manual_seed(2)
    plans = [ta.plan(t.shape) for t in imgs]
    oi, ol = ta.apply(imgs, labs, plans)
    assert oi.shape == (32, 1, 256, 256) and ol.shape == (32, 1, 256, 256) and ol.dtype == torch.int64
    worst = 0.0
    for b, (x, l, p) in enumerate(zip(imgs, labs, plans)):
        noisy = aug._pointwise(x[None, None], aug.OP_NOISE, a=[p["noise_std"]], b=[0.0], seed=p["noise_key"])[0]
        ri, rl = o2.train_branch(noisy[0, 0].cpu().numpy(), l.cpu().numpy(), p["beta"], p["gamma"], p["theta"].numpy(),
                                 p["crop"], [256, 256])
        slack = o2.branch_coordinate_slack(noisy[0, 0].cpu().numpy(), p["beta"], p["gamma"], p["theta"].numpy(),
                                           p["crop"], [256, 256])
        diff = (oi[b, 0].double().cpu().numpy() - ri)
        excess = float((np.abs(diff) - slack).max())
        worst = max(worst, float(np.abs(diff).max()))
        assert excess < TOL, (b, excess)
        assert float(np.median(np.abs(diff))) < 1e-5, b
        assert _mis(ol[b, 0], rl) < LAB_TOL, b
    print("ACDC batch vs fp64 oracle: worst image max abs diff %.2e" % worst)


def test_noise_is_gaussian_noise_bit_for_bit():
    ta = aug.TrainAugment2D([64, 64], **ACDC)
    shapes = [(97, 130), (64, 64), (201, 77)]
    zeros = [torch.zeros(s, device="cuda") for s in shapes]
    labs = [torch.zeros(s, dtype=torch.uint8, device="cuda") for s in shapes]
    y1 = [torch.empty(s, device="cuda") for s in shapes]
    torch.manual_seed(9)
    np.random.seed(9)
    plans = [ta.plan(s) for s in shapes]
    for p in plans:
        p["beta"] = 0.0
    ta.apply(zeros, labs, plans, y1_out=y1)
    for b, (s, p) in enumerate(zip(shapes, plans)):       # what gaussian_noise computes with that key
        ref = aug._pointwise(torch.zeros(1, 1, *s, device="cuda"), aug.OP_NOISE, a=[0.02], b=[0.0], seed=p["noise_key"])[0]
        assert torch.equal(y1[b], ref[0, 0]), b
    torch.manual_seed(9)                                  # and gaussian_noise draws the key the first plan drew
    assert torch.equal(aug.gaussian_noise(torch.zeros(1, 1, *shapes[0], device="cuda"), std=0.02)[0, 0], y1[0])
    assert y1[0].std().item() > 0.015


def test_batch_equals_chain_of_public_functions():
    imgs, labs = _ragged(4, seed=3)
    np.random.seed(4)
    torch.manual_seed(4)
    chain = []
    for x, l in zip(imgs, labs):
        t = aug.gaussian_noise(x[None, None], std=0.02)
        t = aug.brightness_additive(t, std=0.7)
        t = aug.gamma(t, gamma_range=[0.5, 1.6], retain_stats=True)
        t, tl = aug.random_scale_rotate_translate_2d(t, l[None, None], 0.3, 180, 0)
        t, tl = aug.crop_2d(t, tl, [256, 256], mode="random")
        chain.append((t, tl))
    np.random.seed(4)
    torch.manual_seed(4)
    oi, ol = aug.TrainAugment2D([256, 256], **ACDC)(imgs, labs)
    for b, (t, tl) in enumerate(chain):
        assert (oi[b] - t[0]).abs().max().item() < 1e-6, b
        assert torch.equal(ol[b], tl[0]), b


def test_same_plan_same_bits_and_uint8_int64_labels():
    imgs, labs = _ragged(8, seed=5)
    ta = aug.TrainAugment2D([256, 256], **ACDC)
    np.random.seed(6)
    torch.manual_seed(6)
    plans = [ta.plan(t.shape) for t in imgs]
    a_i, a_l = ta.apply(imgs, labs, plans)
    b_i, b_l = ta.apply(imgs, labs, plans)
    c_i, c_l = ta.apply(imgs, [l.long() for l in labs], plans)
    assert torch.equal(a_i, b_i) and torch.equal(a_l, b_l)
    assert torch.equal(a_i, c_i) and torch.equal(a_l, c_l)
    # a slice gives the same bits whatever batch it runs in
    s_i, s_l = ta.apply(imgs[3:4], labs[3:4], plans[3:4])
    assert torch.equal(s_i[0], a_i[3]) and torch.equal(s_l[0], a_l[3])


@pytest.mark.timeout(600)
def test_feeds_one_unet2d_amp_step():
    imgs, labs = _ragged(32, seed=7)
    torch.manual_seed(0)
    np.random.seed(0)
    x, y = aug.TrainAugment2D([256, 256], **ACDC)(imgs, labs)
    net = b200seg.UNet2D(1, 4, 32, block="SingleConv").cuda()
    crit = b200seg.DiceCELoss(weight=torch.tensor([0.5, 1.0, 1.0, 1.0]))
    net.train()
    with torch.autocast("cuda", dtype=torch.float16):
        loss = crit(net(x), y)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item()
    assert all(p.grad is None or torch.isfinite(p.grad).all().item() for p in net.parameters())

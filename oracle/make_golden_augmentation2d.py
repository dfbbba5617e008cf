"""Pin oracle/augmentation2d.py against the UNMODIFIED reference module (training/augmentation.py, 2D branches) and write
tests/golden/augment2d_ops.pt (per-function cases with the random parameters the reference drew: non-square slices,
rotations near +-180 degrees) and tests/golden/augment2d_train.pt (the slice branch of dataset_acdc.py:128-142 driven
with the reference's own functions under fixed np.random seeds, noise std 0).  Runs only where the reference exists.
Usage:  python oracle/make_golden_augmentation2d.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import augmentation2d as o2                       # noqa: E402
from oracle.make_golden_augmentation import import_reference_aug, replay, replay_torch   # noqa: E402

SHAPES = [(70, 90), (97, 64)]
CROP = [48, 48]
CLASSES = 4
BRANCH = dict(scale=0.3, rotate=180, translate=0, gaussian_noise_std=0.0, additive_brightness_std=0.7,
              gamma_range=[0.5, 1.6])


def maxdiff(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max())


def affine_case(ref, img, lab, scale, rotate, translate, seed):
    np.random.seed(seed)
    s0 = np.random.get_state()
    ri, rl = ref.random_scale_rotate_translate_2d(img[None, None], lab[None, None].long(), scale, rotate, translate)
    r6, ang = replay(s0, lambda: o2.draws_affine_2d(scale, rotate, translate))
    theta = o2.theta_from_draws(r6, ang)
    oi, ol = o2.scale_rotate_translate_2d(img[None].numpy(), lab.numpy(), theta)
    d, mis = maxdiff(oi, ri[0]), float((ol != rl[0, 0].numpy()).mean())
    print("affine %s seed %d angle %+4d: image max diff %.2e, label mismatch %.2e" % (list(img.shape), seed, ang, d, mis))
    assert d < 5e-5 and mis < 2e-3
    return {"seed": seed, "args": (scale, rotate, translate), "draws": (r6, ang), "theta": torch.from_numpy(theta.copy()),
            "img": ri[0, 0].clone(), "lab": rl[0, 0].to(torch.uint8)}


def ops_fixture(ref):
    fx = {"crop": CROP, "slices": []}
    for k, (H, W) in enumerate(SHAPES):
        img, lab = o2.make_slice(H, W, CLASSES, seed=500 + k)
        c = {"img": img, "lab": lab, "affine": []}
        # affine: one ordinary draw, then seeds whose angle lands within 5 degrees of +-180
        c["affine"].append(affine_case(ref, img, lab, 0.3, 180, 0.1, seed=3 + 20 * k))
        near = []
        for seed in range(2000):
            np.random.seed(seed)
            _, ang = o2.draws_affine_2d(0.3, 180, 0)
            if abs(ang) >= 175 and (not near or np.sign(ang) != np.sign(near[0][1])):
                near.append((seed, ang))
            if len(near) == 2:
                break
        for seed, _ in near:
            c["affine"].append(affine_case(ref, img, lab, 0.3, 180, 0, seed))
        # crop_2d(random) and (center)
        np.random.seed(40 + k)
        s0 = np.random.get_state()
        ci, cl = ref.crop_2d(img[None, None], lab[None, None], CROP, mode="random")
        org = replay(s0, lambda: [int(np.random.randint(0, max(s - c, 1))) for s, c in zip((H, W), CROP)])
        oi, ol = o2.crop_2d(img[None].numpy(), lab.numpy(), org, CROP)
        assert maxdiff(oi, ci[0]) == 0 and (ol == cl[0, 0].numpy()).all()
        c["crop_seed"], c["crop_origin"], c["crop_img"], c["crop_lab"] = 40 + k, org, ci[0, 0].clone(), cl[0, 0].clone()
        # intensity ops, each with the parameter the reference drew from torch's generator
        x = img[None, None].clone()

        def one(name, call, draw, orc, tol=2e-5):
            ts = torch.get_rng_state()
            y = call(x.clone())
            par = replay_torch(ts, draw)
            d = maxdiff(orc(x[0].numpy(), par), y[0])
            print("%s %-20s param %.6f  max diff %.3e" % ([H, W], name, par, d))
            assert d < tol, name
            c[name] = {"param": par, "out": y[0, 0].clone()}
        torch.manual_seed(60 + k)
        one("brightness_additive", lambda t: ref.brightness_additive(t, std=0.7),
            lambda: float(torch.normal(0, 0.7, size=(1, 1, 1, 1))), lambda a, r: a.astype(np.float64) + r)
        one("brightness_multiply", lambda t: ref.brightness_multiply(t, multiply_range=[0.7, 1.3]),
            lambda: float(torch.rand(size=(1, 1, 1, 1)) * 0.6 + 0.7), lambda a, r: a.astype(np.float64) * r)
        one("gamma", lambda t: ref.gamma(t, gamma_range=[0.5, 1.6], retain_stats=True),
            lambda: float(torch.rand(1, 1) * 1.1 + 0.5), o2.gamma)
        one("gamma_no_retain", lambda t: ref.gamma(t, gamma_range=[0.5, 1.6], retain_stats=False),
            lambda: float(torch.rand(1, 1) * 1.1 + 0.5), lambda a, g: o2.gamma(a, g, retain_stats=False))
        one("contrast", lambda t: ref.contrast(t, contrast_range=[0.65, 1.5]),
            lambda: float(torch.rand(1, 1) * 0.85 + 0.65), o2.contrast)
        one("blur", lambda t: ref.gaussian_blur(t, sigma_range=[0.5, 1.0]), lambda: float(torch.rand(1) * 0.5 + 0.5),
            o2.gaussian_blur)
        for ax in (0, 1):
            assert maxdiff(np.flip(img.numpy(), ax), ref.mirror(img[None, None], axis=ax)[0, 0]) == 0
        fx["slices"].append(c)
    torch.save(fx, os.path.join(ROOT, "tests", "golden", "augment2d_ops.pt"))


def reference_branch(ref, tensor_img, tensor_lab, c):
    """dataset_acdc.py:128-142 statement by statement, on the reference's own functions."""
    tensor_img = tensor_img.unsqueeze(0).unsqueeze(0)
    tensor_lab = tensor_lab.unsqueeze(0).unsqueeze(0)
    tensor_img = ref.gaussian_noise(tensor_img, std=c["gaussian_noise_std"])
    tensor_img = ref.brightness_additive(tensor_img, std=c["additive_brightness_std"])
    tensor_img = ref.gamma(tensor_img, gamma_range=c["gamma_range"], retain_stats=True)
    tensor_img, tensor_lab = ref.random_scale_rotate_translate_2d(tensor_img, tensor_lab, c["scale"], c["rotate"], c["translate"])
    tensor_img, tensor_lab = ref.crop_2d(tensor_img, tensor_lab, CROP, mode="random")
    return tensor_img.squeeze(0), tensor_lab.squeeze(0)


def train_fixture(ref):
    cases = []
    for k, seed in enumerate([7, 8, 9, 10]):
        H, W = SHAPES[k % 2]
        img, lab = o2.make_slice(H, W, CLASSES, seed=600 + k)
        np.random.seed(seed)
        torch.manual_seed(seed)
        s0, t0 = np.random.get_state(), torch.get_rng_state()
        oi, ol = reference_branch(ref, img, lab.long(), BRANCH)

        def torch_draws():
            torch.randn(1, 1, H, W)                       # what gaussian_noise consumed
            beta = float(torch.normal(0, BRANCH["additive_brightness_std"], size=(1, 1, 1, 1)))
            g = float(torch.rand(1, 1) * (BRANCH["gamma_range"][1] - BRANCH["gamma_range"][0]) + BRANCH["gamma_range"][0])
            return beta, g

        def np_draws():
            r6, ang = o2.draws_affine_2d(BRANCH["scale"], BRANCH["rotate"], BRANCH["translate"])
            return r6, ang, [int(np.random.randint(0, max(s - c, 1))) for s, c in zip((H, W), CROP)]
        beta, g = replay_torch(t0, torch_draws)
        r6, ang, crop = replay(s0, np_draws)
        theta = o2.theta_from_draws(r6, ang)
        pi, pl = o2.train_branch(img.numpy(), lab.numpy(), beta, g, theta, crop, CROP)
        d, mis = maxdiff(pi, oi[0]), float((pl != ol[0].numpy()).mean())
        print("branch seed %d %s: beta %+.4f gamma %.4f angle %+4d crop %s  max diff %.2e  label mismatch %.2e"
              % (seed, [H, W], beta, g, ang, crop, d, mis))
        assert d < 5e-5 and mis < 2e-3
        cases.append({"seed": seed, "img_in": img, "lab_in": lab, "beta": beta, "gamma": g, "theta": torch.from_numpy(theta.copy()),
                      "angle": ang, "crop_origin": crop, "img": oi[0].clone(), "lab": ol[0].to(torch.uint8)})
    torch.save({"cfg": dict(BRANCH, training_size=CROP), "cases": cases},
               os.path.join(ROOT, "tests", "golden", "augment2d_train.pt"))


def main():
    torch.set_num_threads(8)
    ref = import_reference_aug()
    ops_fixture(ref)
    train_fixture(ref)


if __name__ == "__main__":
    main()

"""CPU tests of the SSIM / L1+SSIM oracle (oracle_core.h: orc_ssim_forward/backward).

Pins: (1) the textbook definition the reference's own test compares against (fused_ssim/tests/test.py:52-75: depthwise
conv2d with the normalised 11x11 sigma-1.5 window, zero padding) evaluated in float64 with torch, and torch autograd of its
mean for the backward; (2) tests/golden/ssim_small.npz = outputs of the UNMODIFIED reference CUDA kernels on an H100
(tests/golden/make_golden_ssim.py)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle

C1, C2 = 0.01 ** 2, 0.03 ** 2
GAUSS = np.array([0.001028380123898387, 0.0075987582094967365, 0.036000773310661316, 0.10936068743467331, 0.21300552785396576,
                  0.26601171493530273, 0.21300552785396576, 0.10936068743467331, 0.036000773310661316, 0.0075987582094967365,
                  0.001028380123898387], dtype=np.float32).astype(np.float64)      # fused_ssim/ssim.cu:12-24 as fp32


def torch_ssim_map(x, y):
    """fused_ssim/tests/test.py:52-75 with the reference kernel's taps."""
    ch = x.shape[1]
    g = torch.from_numpy(GAUSS)
    win = (g[:, None] * g[None, :])[None, None].expand(ch, 1, 11, 11).contiguous()
    conv = lambda z: F.conv2d(z, win, padding=5, groups=ch)
    mu1, mu2 = conv(x), conv(y)
    s1, s2, s12 = conv(x * x) - mu1 * mu1, conv(y * y) - mu2 * mu2, conv(x * y) - mu1 * mu2
    return ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))


def pair(shape, seed=0):
    rng = np.random.default_rng(seed)
    return rng.random(shape), rng.random(shape)


def test_gaussian_taps_are_the_normalised_sigma_1p5_window():
    g = np.exp(-((np.arange(11) - 5) ** 2) / (2 * 1.5 ** 2))
    assert np.abs(g / g.sum() - GAUSS).max() < 1e-7


@pytest.mark.parametrize("shape", [(2, 3, 37, 53), (1, 1, 1, 1), (1, 2, 5, 70), (1, 3, 64, 32)])
def test_ssim_map_matches_the_conv2d_definition_f64(shape):
    x, y = pair(shape)
    m = oracle.fusedssim(C1, C2, x, y, True)[0]
    want = torch_ssim_map(torch.from_numpy(x), torch.from_numpy(y)).numpy()
    assert np.abs(m - want).max() < 1e-12


@pytest.mark.parametrize("l1", [0, 1])
def test_backward_matches_autograd_of_the_definition_f64(l1):
    x, y = pair((2, 3, 23, 41), seed=3)
    y[0, 0, 2:4, 5:9] = x[0, 0, 2:4, 5:9]                   # ties: sign(0) = 0 (ssim.cu:840)
    up = np.random.default_rng(4).standard_normal(x.shape)
    tx = torch.from_numpy(x).requires_grad_(True)
    ty = torch.from_numpy(y)
    w = 0.2
    smap = torch_ssim_map(tx, ty)
    tmap = w * (1 - smap) + (1 - w) * (tx - ty).abs() if l1 else smap
    (tmap * torch.from_numpy(up)).sum().backward()
    if l1:
        m, d0, d1, d2 = oracle.fusedl1ssim_loss(w, C1, C2, x, y, True)
        g = oracle.fusedl1ssim_loss_backward(w, C1, C2, x, y, up, d0, d1, d2)
    else:
        m, d0, d1, d2 = oracle.fusedssim(C1, C2, x, y, True)
        g = oracle.fusedssim_backward(C1, C2, x, y, up, d0, d1, d2)
    assert np.abs(m - tmap.detach().numpy()).max() < 1e-12
    assert np.abs(g - tx.grad.numpy()).max() < 1e-9 * max(1.0, np.abs(tx.grad.numpy()).max())


def test_f32_oracle_tracks_f64_and_train_false_returns_empty_partials():
    x, y = pair((1, 3, 40, 60), seed=5)
    m64, a64, b64, c64 = oracle.fusedssim(C1, C2, x, y, True)
    m32, a32, b32, c32 = oracle.fusedssim(C1, C2, x.astype(np.float32), y.astype(np.float32), True)
    for u, v in ((m32, m64), (a32, a64), (b32, b64), (c32, c64)):
        assert np.abs(u - v).max() <= 2e-5 * max(1.0, np.abs(v).max())
    m, a, b, c = oracle.fusedssim(C1, C2, x, y, False)
    assert a.size == 0 and b.size == 0 and c.size == 0 and np.array_equal(m, m64)


GOLD = os.path.join(os.path.dirname(__file__), "golden", "ssim_small.npz")


@pytest.mark.parametrize("name", ["rand", "smooth"])
@pytest.mark.parametrize("mode", ["ssim", "l1"])
def test_oracle_matches_reference_cuda_golden(name, mode):
    """The reference kernels run in fp32 with --use_fast_math; the fp64 oracle must agree to fp32 rounding: 1e-4 on the
    random pair, and on the smooth pair (sigma = E[x^2] - mu^2 cancels, B = sigma1 + sigma2 + C2 ~ 1e-3) to 4x what the
    oracle's own fp32 instantiation loses against fp64 on that input."""
    from tests.golden.make_golden_ssim import inputs
    z = np.load(GOLD)
    pairs, up = inputs()
    x, y, up = pairs[name][0].astype(np.float64), pairs[name][1].astype(np.float64), up.astype(np.float64)
    c1, c2, w = float(z["C1"]), float(z["C2"]), float(z["ssim_weight"])
    if mode == "l1":
        m, d0, d1, d2 = oracle.fusedl1ssim_loss(w, c1, c2, x, y, True)
        g = oracle.fusedl1ssim_loss_backward(w, c1, c2, x, y, up, d0, d1, d2)
    else:
        m, d0, d1, d2 = oracle.fusedssim(c1, c2, x, y, True)
        g = oracle.fusedssim_backward(c1, c2, x, y, up, d0, d1, d2)
    x32, y32, up32 = x.astype(np.float32), y.astype(np.float32), up.astype(np.float32)
    if mode == "l1":
        f = oracle.fusedl1ssim_loss(w, c1, c2, x32, y32, True)
        f = f + (oracle.fusedl1ssim_loss_backward(w, c1, c2, x32, y32, up32, f[1], f[2], f[3]),)
    else:
        f = oracle.fusedssim(c1, c2, x32, y32, True)
        f = f + (oracle.fusedssim_backward(c1, c2, x32, y32, up32, f[1], f[2], f[3]),)
    for k, v, v32 in zip(("map", "dm_dmu1", "dm_dsigma1_sq", "dm_dsigma12", "grad"), (m, d0, d1, d2, g), f):
        ref = z[f"{name}_{mode}_{k}"]
        scale = max(1.0, np.abs(ref).max())
        err = np.abs(v - ref).max() / scale
        cond = np.abs(v32.astype(np.float64) - v).max() / scale
        bound = max(1e-4, 4.0 * cond)
        if name == "rand":
            assert bound == 1e-4
        assert err < bound, (k, err, cond)

"""TEST INFRASTRUCTURE -- information-weighted multi-scale SSIM (IW-SSIM, Wang & Li 2011) as src/evaluate.py:81-88 reports
it through src/util/IW_SSIM_PyTorch.py with its default parameters, restated in torch for any device and dtype.

Every stage is exposed, so that a comparison can find the stage where two computations part:
    evaluate_gray   rgb2gray(x.view(W, H, -1)) of evaluate.py:57-61 (fp32 arithmetic, round half to even);
    bands           the Laplacian pyramid (oracle/laplacian_pyramid.py, float64), rounded once to `dtype`;
    quality_maps    cs maps of every scale and the l map of the last, from valid 11x11 Gaussian statistics;
    info_weights    the information-content weight maps of scales 1-4 (3x3 neighbourhoods plus the parent band);
    iwssim          all of it: dict(bands, cs, l, iw, wmcs, score).
The original (reference) image weights the scales and supplies the parent band; the distorted one is the image under test.
A scale whose rebuilt covariance cannot be inverted gets NaN (where the reference's torch.inverse raises).
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.laplacian_pyramid import laplacian_pyramid

NSC = 5
K = (0.01, 0.03)
L = 255
# the scale weights (0.0448, 0.2856, 0.3001, 0.2363, 0.1333) as the reference holds them: a default-dtype (fp32) tensor,
# widened afterwards, so even its fp64 path raises the wmcs to the fp32-rounded weights
WEIGHTS = tuple(float(w) for w in np.array([0.0448, 0.2856, 0.3001, 0.2363, 0.1333], np.float32))
WINSIZE, SIGMA = 11, 1.5
BLOCK = 3                 # 3 x 3 neighbourhoods
SIGMA_NSQ = 0.4
TOL = 1e-15
BOUND1 = 4                # ceil((11 - 1) / 2) - floor((3 - 1) / 2): the crop that aligns an iw map with its cs map
MIN_SIZE = 161            # the coarsest band, ceil(n / 16), must hold one 11 x 11 window


def evaluate_gray(x, W, H):
    """evaluate.py's rgb2gray(x.view(W, H, -1)): [H*W, 3] fp32 -> [W, H] fp32 of rounded gray values."""
    v = x.to(torch.float32).reshape(W, H, 3)
    gray = 0.2989 * v[:, :, 0] + 0.5870 * v[:, :, 1] + 0.1140 * v[:, :, 2]
    return torch.round(gray)


def gaussian_window(dtype=torch.float64, device="cpu"):
    r = WINSIZE // 2
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    g = np.exp(-(x ** 2 + y ** 2) / (2.0 * SIGMA ** 2))
    g[g < np.finfo(g.dtype).eps * g.max()] = 0
    g /= g.sum()
    return torch.from_numpy(g)[None, None].to(device=device, dtype=dtype)


def bands(image, dtype=torch.float64, device="cpu"):
    """The 5 pyramid entries of a 2-D image, computed in float64 and rounded once to dtype, as [1, 1, h, w] tensors."""
    im = image.detach().cpu().double().numpy() if torch.is_tensor(image) else np.asarray(image, np.float64)
    return [torch.from_numpy(b)[None, None].to(device=device, dtype=dtype) for b in laplacian_pyramid(im, NSC)]


def quality_maps(bo, bd):
    """(cs maps of scales 1..5, l map of scale 5) from valid 11 x 11 Gaussian statistics."""
    win = gaussian_window(bo[0].dtype, bo[0].device)
    C1, C2 = (K[0] * L) ** 2, (K[1] * L) ** 2
    cs = []
    for x, y in zip(bo, bd):
        mu1, mu2 = F.conv2d(x, win), F.conv2d(y, win)
        s12 = F.conv2d(x * y, win) - mu1 * mu2
        s1 = torch.clamp_min(F.conv2d(x * x, win) - mu1 * mu1, 0)
        s2 = torch.clamp_min(F.conv2d(y * y, win) - mu2 * mu2, 0)
        cs.append((2 * s12 + C2) / (s1 + s2 + C2))
    return cs, (2 * mu1 * mu2 + C1) / (mu1 ** 2 + mu2 ** 2 + C1)


def enlarge2(im):
    """The parent band on its child's grid: bilinear to (4M - 3, 4N - 3), the border extrapolated linearly (rows, then
    columns), every other sample -> [1, 1, 2M, 2N]."""
    _, _, M, N = im.shape
    t1 = F.interpolate(im, size=(4 * M - 3, 4 * N - 3), mode="bilinear", align_corners=False)
    t2 = torch.zeros((1, 1, 4 * M - 1, 4 * N - 1), dtype=im.dtype, device=im.device)
    t2[:, :, 1:-1, 1:-1] = t1
    t2[:, :, 0, :] = 2 * t2[:, :, 1, :] - t2[:, :, 2, :]
    t2[:, :, -1, :] = 2 * t2[:, :, -2, :] - t2[:, :, -3, :]
    t2[:, :, :, 0] = 2 * t2[:, :, :, 1] - t2[:, :, :, 2]
    t2[:, :, :, -1] = 2 * t2[:, :, :, -2] - t2[:, :, :, -3]
    return t2[:, :, ::2, ::2]


def neighbourhood_vectors(bo, s):
    """Y [n_interior, 9 (+ 1)]: each interior pixel's 3 x 3 neighbours in the original band s (0-based), plus its parent
    at s < NSC - 2."""
    x = bo[s][0, 0]
    nv, nh = x.shape
    cols = [x[1 + dy:nv - 1 + dy, 1 + dx:nh - 1 + dx].reshape(-1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    if s < NSC - 2:
        cols.append(enlarge2(bo[s + 1])[0, 0, 1:nv - 1, 1:nh - 1].reshape(-1))
    return torch.stack(cols, 1)


def covariance_inverse(C):
    """(raw eigenvalues, inverse of the covariance rebuilt with negative eigenvalues zeroed and the positive ones rescaled
    to keep their sum), or NaNs where the rebuilt matrix cannot be inverted."""
    lam, V = torch.linalg.eigh(C)
    pos = lam * (lam > 0).to(lam.dtype)
    sp = pos.sum()
    Ladj = torch.diag(pos) * lam.sum() / (sp + (sp == 0).to(lam.dtype))
    R = V @ Ladj @ V.T
    inv, info = torch.linalg.inv_ex(R)
    if info.item() != 0 or not bool(torch.isfinite(inv).all()):
        inv = torch.full_like(R, float("nan"))
    return lam, inv


def info_weights(bo, bd):
    """iw maps of scales 1..4, cropped by BOUND1 so that each lines up with its cs map."""
    dt, dev = bo[0].dtype, bo[0].device
    box = torch.full((1, 1, BLOCK, BLOCK), 1.0 / (BLOCK * BLOCK), dtype=torch.float64).to(device=dev, dtype=dt)
    iw = []
    for s in range(NSC - 1):
        x, y = bo[s], bd[s]
        mx, my = F.conv2d(x, box, padding=1), F.conv2d(y, box, padding=1)
        cxy = F.conv2d(x * y, box, padding=1) - mx * my
        sx = F.conv2d(x * x, box, padding=1) - mx ** 2
        sy = F.conv2d(y * y, box, padding=1) - my ** 2
        sx = torch.where(sx < 0, torch.zeros_like(sx), sx)
        sy = torch.where(sy < 0, torch.zeros_like(sy), sy)
        g = cxy / (sx + TOL)
        vv = sy - g * cxy
        g = torch.where(sx < TOL, torch.zeros_like(g), g)
        vv = torch.where(sx < TOL, sy, vv)
        g = torch.where(sy < TOL, torch.zeros_like(g), g)
        vv = torch.where(sy < TOL, torch.zeros_like(vv), vv)
        Y = neighbourhood_vectors(bo, s)
        n, N = Y.shape
        lam, Cinv = covariance_inverse(Y.T @ Y / n)
        nv, nh = x.shape[2] - 2, x.shape[3] - 2
        ss = ((Y @ Cinv) * Y).sum(1).view(1, 1, nv, nh) / N
        g, vv = g[:, :, 1:-1, 1:-1], vv[:, :, 1:-1, 1:-1]
        w = torch.zeros_like(g)
        for lj in lam:
            w = w + torch.log2(1 + ((vv + (1 + g * g) * SIGMA_NSQ) * ss * lj + SIGMA_NSQ * vv) / (SIGMA_NSQ * SIGMA_NSQ))
        w = torch.where(w < TOL, torch.zeros_like(w), w)
        iw.append(w[:, :, BOUND1:-BOUND1, BOUND1:-BOUND1])
    return iw


def iwssim(original, distorted, dtype=torch.float64, device=None):
    """IW-SSIM of `distorted` against `original` (2-D images on the metric's scale): every stage and the score."""
    device = device if device is not None else (original.device if torch.is_tensor(original) else "cpu")
    bo, bd = bands(original, dtype, device), bands(distorted, dtype, device)
    cs, lmap = quality_maps(bo, bd)
    iw = info_weights(bo, bd)
    wmcs = [float((cs[s] * iw[s]).sum() / iw[s].sum()) for s in range(NSC - 1)]
    wmcs.append(float((cs[-1] * lmap).mean()))
    score = float(np.prod(np.abs(np.array(wmcs, np.float64)) ** np.array(WEIGHTS, np.float64)))
    return dict(bands=(bo, bd), cs=cs, l=lmap, iw=iw, wmcs=wmcs, score=score)


def metric_images(image, reference, W, H, layout):
    """(original, distorted) 2-D images the metric sees for adn_image_iwssim's inputs: the reference is the original."""
    if layout == "evaluate":
        return evaluate_gray(reference, W, H), evaluate_gray(image, W, H)
    return reference.to(torch.float32).reshape(H, W), image.to(torch.float32).reshape(H, W)

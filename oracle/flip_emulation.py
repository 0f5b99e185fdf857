"""TEST INFRASTRUCTURE -- FLIP (Andersson et al., HPG 2020) as src/evaluate.py:119-161 evaluates it, restated in torch from
the metric's definition: the same code runs on any device and in any dtype (fp64 on the CPU for the golden checks, fp64 on
the GPU at frame size, fp32 on the GPU as the benchmark's baseline).

It applies every filter as the full 2-D kernel the definition gives (conv2d over a replicate-padded image), not as the
1-D factors adn_image_flip uses, so agreement also checks that factorisation.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

EVALUATE_PPD = 0.7 * (3840 / 0.7) * (np.pi / 180)
QC, QF, PC, PT = 0.7, 0.5, 0.4, 0.95

# linear RGB -> CIE XYZ under D65 (exact rationals); the white point is its row sums
RGB2XYZ = np.array([[10135552 / 24577794, 8788810 / 24577794, 4435075 / 24577794],
                    [2613072 / 12288897, 8788810 / 12288897, 887015 / 12288897],
                    [1425312 / 73733382, 8788810 / 73733382, 70074185 / 73733382]])
# contrast sensitivity of the three opponent channels: (a1, b1, a2, b2) of a1 sqrt(pi/b1) exp(-pi^2 z/b1) + a2 sqrt(pi/b2) exp(..)
CSF = {"A": (1.0, 0.0047, 0.0, 1e-5), "RG": (1.0, 0.0053, 0.0, 1e-5), "BY": (34.1, 0.04, 13.5, 0.025)}


def csf_radius(ppd):
    return int(math.ceil(3 * math.sqrt(0.04 / (2 * math.pi ** 2)) * ppd))


def feature_radius(ppd):
    return int(math.ceil(3 * 0.5 * 0.082 * ppd))


def csf_kernel(ppd, channel):
    """[2r+1, 2r+1] float64, normalised to sum 1."""
    a1, b1, a2, b2 = CSF[channel]
    r = csf_radius(ppd)
    t = np.arange(-r, r + 1) / ppd
    z = t[None, :] ** 2 + t[:, None] ** 2
    g = a1 * np.sqrt(np.pi / b1) * np.exp(-np.pi ** 2 * z / b1) + a2 * np.sqrt(np.pi / b2) * np.exp(-np.pi ** 2 * z / b2)
    return g / g.sum()


def feature_kernel(ppd, kind):
    """The x-direction edge (first derivative) or point (second derivative) detector, [2r+1, 2r+1] float64: positive
    weights scaled to sum 1, negative ones to sum -1."""
    sd = 0.5 * 0.082 * ppd
    r = feature_radius(ppd)
    x, y = np.meshgrid(np.arange(-r, r + 1), np.arange(-r, r + 1))
    g = np.exp(-(x ** 2 + y ** 2) / (2 * sd * sd))
    k = -x * g if kind == "edge" else (x ** 2 / (sd * sd) - 1) * g
    return np.where(k < 0, k / -k[k < 0].sum(), k / k[k > 0].sum())


def _mat(m, img):
    return torch.einsum("ij,njhw->nihw", torch.as_tensor(m, dtype=img.dtype, device=img.device), img)


def _white():
    return RGB2XYZ.sum(1)


def srgb_to_ycxcz(img):
    c = torch.clamp(img, 0.0, 1.0)
    lin = torch.where(c > 0.04045, torch.pow((c + 0.055) / 1.055, 2.4), c / 12.92)
    xyz = _mat(RGB2XYZ / _white()[:, None], lin)
    return torch.cat([116 * xyz[:, 1:2] - 16, 500 * (xyz[:, 0:1] - xyz[:, 1:2]), 200 * (xyz[:, 1:2] - xyz[:, 2:3])], 1)


def ycxcz_to_linrgb(img):
    y = (img[:, 0:1] + 16) / 116
    xyz = torch.cat([y + img[:, 1:2] / 500, y, y - img[:, 2:3] / 200], 1)
    return _mat(np.linalg.inv(RGB2XYZ) * _white()[None, :], xyz)


def linrgb_to_hunt_lab(lin):
    t = _mat(RGB2XYZ / _white()[:, None], lin)
    d = 6 / 29
    f = torch.where(t > 0.00885, torch.pow(t, 1 / 3), t / (3 * d * d) + 4 / 29)
    L = 116 * f[:, 1:2] - 16
    return torch.cat([L, 0.01 * L * (500 * (f[:, 0:1] - f[:, 1:2])), 0.01 * L * (200 * (f[:, 1:2] - f[:, 2:3]))], 1)


def hyab(p, q):
    d = p - q
    return torch.abs(d[:, 0:1]) + torch.sqrt(d[:, 1:2] ** 2 + d[:, 2:3] ** 2)


def cmax(dtype=torch.float64):
    rgb = torch.tensor([[0.0, 1.0, 0.0], [0.0, 0.0, 1.0]], dtype=dtype).reshape(2, 3, 1, 1)
    lab = linrgb_to_hunt_lab(rgb)
    return float(torch.pow(hyab(lab[0:1], lab[1:2]), QC))


def _conv(img, kernel):
    k = torch.as_tensor(kernel, dtype=img.dtype, device=img.device)[None, None]
    r = kernel.shape[0] // 2
    return F.conv2d(F.pad(img, (r, r, r, r), mode="replicate"), k)


def flip_map(image, reference, W, H, ppd=EVALUATE_PPD, dtype=torch.float64):
    """image, reference: [H*W, 3] or [H, W, 3] sRGB tensors (any device) -> the FLIP map [H, W] in `dtype` on that device."""
    imgs = [t.reshape(H, W, 3).permute(2, 0, 1)[None].to(dtype) for t in (image, reference)]
    ycc = [srgb_to_ycxcz(t) for t in imgs]
    # colour: CSF-filtered opponent channels, back to linear RGB clamped to the box, Hunt-adjusted L*a*b*, HyAB
    kern = [csf_kernel(ppd, ch) for ch in ("A", "RG", "BY")]
    lab = [linrgb_to_hunt_lab(torch.clamp(ycxcz_to_linrgb(torch.cat([_conv(t[:, i:i + 1], kern[i]) for i in range(3)], 1)),
                                          0.0, 1.0)) for t in ycc]
    p = torch.pow(hyab(lab[0], lab[1]), QC)
    cm = cmax(dtype)
    pccmax = PC * cm
    dec = torch.where(p < pccmax, (PT / pccmax) * p, PT + ((p - pccmax) / (cm - pccmax)) * (1.0 - PT))
    # features: edge and point magnitudes of the normalised unfiltered luminance
    edge, point = feature_kernel(ppd, "edge"), feature_kernel(ppd, "point")
    mags = []
    for t in ycc:
        y = (t[:, 0:1] + 16) / 116
        mags.append([torch.sqrt(_conv(y, k) ** 2 + _conv(y, k.T) ** 2) for k in (edge, point)])
    df = torch.maximum(torch.abs(mags[0][0] - mags[1][0]), torch.abs(mags[0][1] - mags[1][1]))
    def_ = torch.clamp(torch.pow(df / math.sqrt(2), QF), 0.0, 1.0)
    return torch.pow(dec, 1 - def_)[0, 0]


def flip(image, reference, W, H, ppd=EVALUATE_PPD, dtype=torch.float64):
    """-> (map [H, W], mean as a Python float)."""
    m = flip_map(image, reference, W, H, ppd, dtype)
    return m, float(m.mean())

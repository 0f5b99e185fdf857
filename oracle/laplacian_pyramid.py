"""TEST INFRASTRUCTURE -- the Laplacian pyramid IW-SSIM builds its scales from (pyrtools' LaplacianPyramid(img, height)
with its defaults), restated in numpy float64.

    filter   binom5 = sqrt(2) * [1, 4, 6, 4, 1] / 16, applied along rows and along columns (not normalised: each
             reduction multiplies a constant by 2);
    corrDn   reflect-pad the signal by 2 about its edge sample (numpy "reflect": x[-1] = x[1]), correlate, keep every
             other sample from index 0 -> ceil(n / 2) samples;
    upConv   zero-insert the coarse signal onto the output grid (sample k at 2k), reflect-pad that signal the same way,
             correlate;
    bands    band l = level l - upConv(level l + 1), l < height - 1; the last entry is the low-pass level itself.

The edge rule of upConv is this project's restatement ("reflect1" in pyrtools): with it a constant image gives zero bands
and a low-pass of 2^(height-1) times the constant.  The fixtures under tests/golden/iwssim_* pin this restatement.
"""
import numpy as np

BINOM5 = np.sqrt(2.0) * np.array([1.0, 4.0, 6.0, 4.0, 1.0]) / 16.0


def _correlate(x, axis):
    """Correlate along `axis` with BINOM5 after reflect-padding by 2 (the output has the input's length)."""
    pad = [(0, 0)] * x.ndim
    pad[axis] = (2, 2)
    xp = np.pad(x, pad, mode="reflect")
    n = x.shape[axis]
    out = np.zeros_like(x)
    for k, w in enumerate(BINOM5):
        out += w * np.take(xp, np.arange(k, k + n), axis=axis)
    return out


def corr_dn(x, axis):
    return np.take(_correlate(x, axis), np.arange(0, x.shape[axis], 2), axis=axis)


def up_conv(x, axis, n):
    shape = list(x.shape)
    shape[axis] = n
    z = np.zeros(shape)
    idx = [slice(None)] * x.ndim
    idx[axis] = slice(0, n, 2)
    z[tuple(idx)] = x
    return _correlate(z, axis)


def reduce(im):
    return corr_dn(corr_dn(im, 0), 1)


def expand(im, shape):
    return up_conv(up_conv(im, 0, shape[0]), 1, shape[1])


def laplacian_pyramid(image, height=5):
    """[band 0, ..., band height-2, low-pass] in float64; band l is ceil(n / 2^l) in each dimension."""
    im = np.asarray(image, np.float64)
    bands = []
    for _ in range(height - 1):
        nxt = reduce(im)
        bands.append(im - expand(nxt, im.shape))
        im = nxt
    bands.append(im)
    return bands


def reconstruct(bands):
    im = bands[-1]
    for b in reversed(bands[:-1]):
        im = b + expand(im, b.shape)
    return im

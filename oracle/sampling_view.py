"""numpy emulation of the sampling network's view (the C++ viewer's render-oracle mode, samplesToImage in
adanerf_real_time_viewer/src/cuda/base_cuda_kernels.cu:487-528) and of our sampling_view_kernel (stages.cu), bit for bit.

Per ray the viewer sorts the 128 (raw0 value, cell) pairs with cub::BlockRadixSort<float, 128, 1, int>::SortDescending and
draws the first three cells c0, c1, c2 as uchar4(clamp((c + 0.5) / 128, 0, 1) * 255, ..., 255).  The radix sort orders the
twiddled bit patterns of the keys and is stable; the CUB of CUDA 12.x maps -0 to +0 before ranking
(cub/block/radix_rank_sort_operations.cuh, ProcessFloatMinusZero).  So a positive NaN ranks above +inf, a negative NaN
below -inf, and equal keys keep the lower cell first."""
import numpy as np

F32 = np.float32


def keys(raw0):
    """The order-preserving uint32 keys of raw0 [..., 128] (CUB's twiddle, -0 ranked as +0)."""
    b = np.ascontiguousarray(raw0, dtype=F32).view(np.uint32)
    k = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return np.where(k == np.uint32(0x7FFFFFFF), np.uint32(0x80000000), k).astype(np.uint32)


def top3(raw0):
    """[N, 3] int64: the first three cells of each row's stable descending key order."""
    k = keys(np.asarray(raw0, dtype=F32).reshape(-1, 128)).astype(np.uint64)
    cell = np.arange(128, dtype=np.uint64)
    comp = (k << np.uint64(7)) | (np.uint64(127) - cell)          # unique per row: key descending, then cell ascending
    part = np.argpartition(comp, 125, axis=1)[:, 125:]              # the three largest, unordered
    order = np.argsort(np.take_along_axis(comp, part, axis=1), axis=1)[:, ::-1]
    return np.take_along_axis(part, order, axis=1).astype(np.int64)


def sampling_view(raw0):
    """raw0 [N, 128] -> (rgb [N, 3] float32 = (c + 0.5) / 128, rgba8 [N, 4] uint8 = clamp(v, 0, 1) * 255 truncated, 255)."""
    c = top3(raw0)
    rgb = (F32(0.5) + c.astype(F32)) / F32(128.0)
    px = np.empty((c.shape[0], 4), np.uint8)
    px[:, :3] = (np.clip(rgb, F32(0), F32(1)) * F32(255.0)).astype(np.uint8)
    px[:, 3] = 255
    return rgb.astype(F32), px

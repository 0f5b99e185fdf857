"""Image-tile sharding across GPUs (SURVEY.md 8e): rays are independent, so a frame is split into contiguous
row bands (ray id = y*W + x), every rank renders its band with the same kernels and replicated weights, and ONE
collective per frame gathers the RGB tiles.  No other exchange exists on this path."""
import torch
import torch.distributed as dist


def row_bands(H, world_size):
    """[(row0, rows)] per rank; bands differ by at most one row and cover [0, H) in rank order."""
    base, extra = divmod(H, world_size)
    out, r0 = [], 0
    for r in range(world_size):
        rows = base + (1 if r < extra else 0)
        out.append((r0, rows))
        r0 += rows
    return out


def gather_bands(band, W, H, group=None, dst=None):
    """band: this rank's [rows*W, C] tile.  Returns the full [H*W, C] frame on every rank (dst=None, all-gather)
    or on rank `dst` only (gather; other ranks get None).  Equal bands use all_gather_into_tensor (one NCCL
    collective over NVLink); ragged bands are padded to the largest band."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    bands = row_bands(H, world)
    C = band.shape[1]
    max_rows = max(b[1] for b in bands)
    equal = all(b[1] == max_rows for b in bands)
    if equal and dst is None:
        full = torch.empty((H * W, C), dtype=band.dtype, device=band.device)
        dist.all_gather_into_tensor(full, band.contiguous(), group=group)
        return full
    pad = band
    if band.shape[0] != max_rows * W:
        pad = torch.zeros((max_rows * W, C), dtype=band.dtype, device=band.device)
        pad[:band.shape[0]] = band
    if dst is None:
        parts = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(parts, pad.contiguous(), group=group)
    else:
        parts = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
        dist.gather(pad.contiguous(), parts, dst=dst, group=group)
        if rank != dst:
            return None
    return torch.cat([p[:rows * W] for p, (_, rows) in zip(parts, bands)], 0)


def render_frame_distributed(renderer, pose, rot, W, H, thr, K, group=None, dst=None, sample_budget=None):
    """Each rank renders its row band (adn_render_camera with row0/rows) and the tiles are gathered.

    sample_budget=B: at most B samples in the whole frame, every band at the one threshold a single renderer would choose
    for the frame (the gathered frame equals its budgeted frame bit for bit).  The ranks' renderers form a budget group
    whose reducer is dist.all_reduce(SUM) over `group`, for this call; afterwards the renderer has no budget and no group.
    Every rank checks the budget against the frame before anything is enqueued, so all ranks refuse the same frames."""
    rank = dist.get_rank(group)
    row0, rows = row_bands(H, dist.get_world_size(group))[rank]
    if sample_budget is None:
        band = renderer.render_camera(pose, rot, W, H, thr, K, row0=row0, rows=rows)["rgb"]
        return gather_bands(band, W, H, group=group, dst=dst)
    B = int(sample_budget)
    if not thr > 0:
        raise ValueError("render_frame_distributed: sample_budget needs the adaptive path (thr > 0), not dense mode")
    if B < W * H:
        raise ValueError(f"render_frame_distributed: sample_budget {B} is below the {W * H} rays of the frame")
    if W * H * (K - 1) >= 1 << 32:
        raise ValueError("render_frame_distributed: sample_budget supports at most 2^32 - 1 candidate samples (W * H * (K - 1))")
    renderer.set_option("sample_budget", B)
    renderer.set_budget_group(lambda words: dist.all_reduce(words, op=dist.ReduceOp.SUM, group=group))
    try:
        band = renderer.render_camera(pose, rot, W, H, thr, K, row0=row0, rows=rows)["rgb"]
    finally:
        renderer.set_budget_group(None)
        renderer.set_option("sample_budget", 0)
    return gather_bands(band, W, H, group=group, dst=dst)

"""Issue order across streams for the views entries (adn_render_views_rays, adn_render_views_camera,
adn_render_views_camera_rgba8), with the gate and the serial references of tests/test_stream_order.py: a views call on s2
runs only after a full-frame render held on s1, and records the order the next call waits on.  Also the coverage check
over every stream entry include/adanerf_b200_views.h declares."""
import ctypes as C

import numpy as np
import pytest
import torch

import test_stream_order as so
from test_stream_order import gate, shaped   # noqa: F401  (module fixtures)

V = 2
N_PER_VIEW = so.N_RAYS // V
CAM_W, CAM_H = 200, 50                      # V frames of 10 000 rays: the 20 000 rays of the single-view entries


def _tables(e):
    """Two views: the context's camera and one moved and turned, as [V,3] / [V,9] host arrays."""
    poses = np.stack([e.pose, e.pose + np.float32([0.02, -0.01, 0.015])]).astype(np.float32)
    rots = np.stack([e.rot, e.rot.reshape(3, 3)[[1, 0, 2]].reshape(9)]).astype(np.float32)
    return np.ascontiguousarray(poses), np.ascontiguousarray(rots)


def _o_views_rays(e):
    return dict(rgb=so._dev((so.N_RAYS, 3)), n_samples=so._dev((so.N_RAYS,), torch.int32), **so._aux_outputs(so.N_RAYS, e.K))


def _c_views_rays(e, st, o):
    p, r = _tables(e)
    return e.lib.adn_render_views_rays(e.h, V, so._fp(p), so._fp(r), e.dirs.data_ptr(), N_PER_VIEW, e.thr, e.K, o["rgb"].data_ptr(),
                                       o["n_samples"].data_ptr(), None, C.byref(so._aux(o)), C.c_void_p(st))


def _o_views_camera(e):
    return dict(rgb=so._dev((V * CAM_W * CAM_H, 3)), n_samples=so._dev((V * CAM_W * CAM_H,), torch.int32))


def _c_views_camera(e, st, o):
    p, r = _tables(e)
    return e.lib.adn_render_views_camera(e.h, V, so._fp(p), so._fp(r), CAM_W, CAM_H, e.thr, e.K, o["rgb"].data_ptr(),
                                         o["n_samples"].data_ptr(), C.c_void_p(st))


def _o_views_camera_rgba8(e):
    return dict(rgba8=so._dev((V * CAM_W * CAM_H, 4), torch.uint8))


def _c_views_camera_rgba8(e, st, o):
    p, r = _tables(e)
    return e.lib.adn_render_views_camera_rgba8(e.h, V, so._fp(p), so._fp(r), CAM_W, CAM_H, e.thr, e.K, o["rgba8"].data_ptr(),
                                               C.c_void_p(st))


VIEWS_ENTRY_POINTS = {
    "adn_render_views_rays": (_c_views_rays, _o_views_rays),
    "adn_render_views_camera": (_c_views_camera, _o_views_camera),
    "adn_render_views_camera_rgba8": (_c_views_camera_rgba8, _o_views_camera_rgba8),
}


def _case(name):
    call, outputs = VIEWS_ENTRY_POINTS[name]
    return name, call, outputs


VIEWS_HEADER = so.HEADER.replace("adanerf_b200.h", "adanerf_b200_views.h")


def views_header_entries():
    """The functions include/adanerf_b200_views.h declares with a `void* stream` parameter (test_stream_order's rule)."""
    import re
    with open(VIEWS_HEADER) as fh:
        text = re.sub(r"/\*.*?\*/", "", fh.read(), flags=re.S)
    return {name for name, args in re.findall(r"adn_status\s+(adn_\w+)\s*\(([^;]*)\)\s*;", text)
            if re.search(r"void\s*\*\s*stream\b", args) or name.endswith("_host")}


def test_every_views_stream_entry_point_is_covered():
    """A new views entry point with a stream cannot skip the ordering tests: every one include/adanerf_b200_views.h
    declares is gated here (tests/test_stream_order.py gates those of include/adanerf_b200.h)."""
    names = views_header_entries()
    assert names == set(VIEWS_ENTRY_POINTS), (sorted(names ^ set(VIEWS_ENTRY_POINTS)))
    assert not names & so.header_entries()


@pytest.mark.gpu
@pytest.mark.parametrize("s1_kind", ["legacy", "side"])
@pytest.mark.parametrize("b_name", sorted(VIEWS_ENTRY_POINTS))
def test_views_call_waits(shaped, gate, s1_kind, b_name):   # noqa: F811
    """A full-frame render held at the gate on s1, then the views entry on s2: it runs only after the render, and both
    equal their serial references (the views entries launch stage 2, so both sides are first paired with a partner that
    launches none)."""
    with so._options(shaped, chunk_rays=50_000):
        so._ordered_pair(shaped, gate, so._stream(gate, s1_kind), ("render_camera 800x800 K16", so._c_frame, so._o_frame),
                         _case(b_name), True, True)


@pytest.mark.gpu
@pytest.mark.parametrize("a_name", sorted(VIEWS_ENTRY_POINTS))
def test_views_call_orders_the_next(shaped, gate, a_name):   # noqa: F811
    """The views entry as A on gated s1, then a budgeted render as B on s2: the views call records the order B waits on."""
    so._ordered_pair(shaped, gate, gate.s1, _case(a_name), ("render_rays budget K16", so._c_budgeted, so._o_budgeted), True, True)

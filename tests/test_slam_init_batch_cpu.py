"""ovb_slam_delayed_init_batch refuses malformed arguments before it touches a device (no context, no frame, no quaternions,
no output arrays)."""
import ctypes as C

import numpy as np
import pytest

from open_vins_b200 import capi


@pytest.fixture(scope="module")
def lib():
    from open_vins_b200 import build
    build.build()
    return capi.load_library()


def test_malformed_arguments_are_refused_without_a_device(lib):
    fr, fb, op = capi.ovb_frame(), capi.ovb_feat_batch(), capi.default_opts()
    cq, kq = np.zeros((1, 4)), np.zeros((1, 4))
    quat = capi.ovb_frame_quat(cq.ctypes.data_as(capi.c_double_p), kq.ctypes.data_as(capi.c_double_p))
    out = capi.FeatOut(1)
    lm, dxn, dx = np.zeros(1, dtype=np.int32), np.zeros((1, 3)), np.zeros((1, 8))
    ptrs = dict(lm=lm.ctypes.data_as(capi.c_int_p), dxn=dxn.ctypes.data_as(capi.c_double_p), dx=dx.ctypes.data_as(capi.c_double_p))
    fake_ctx = C.c_void_p(8)  # never dereferenced: every call below lacks a required argument and must return before using it

    def call(ctx=fake_ctx, frame=C.byref(fr), q=C.byref(quat), o=C.byref(out.struct()), lm_=ptrs["lm"], dxn_=ptrs["dxn"], dx_=ptrs["dx"]):
        return lib.ovb_slam_delayed_init_batch(ctx, frame, q, C.byref(fb), C.byref(op), None, None, None, o, lm_, dxn_, dx_, 8)
    assert call(ctx=None) == capi.OVB_ERR_ARG
    assert call(frame=None) == capi.OVB_ERR_ARG
    assert call(q=None) == capi.OVB_ERR_ARG
    assert call(q=C.byref(capi.ovb_frame_quat(None, None))) == capi.OVB_ERR_ARG
    assert call(o=None) == capi.OVB_ERR_ARG
    assert call(lm_=None) == capi.OVB_ERR_ARG
    assert call(dxn_=None) == capi.OVB_ERR_ARG
    assert call(dx_=None) == capi.OVB_ERR_ARG

"""CPU test of the C-ABI's argument checking: malformed descriptors are refused with EMO_ERR_INVALID and a message
BEFORE anything is launched (so this runs without a GPU; no compute call is made — every call below fails its guard)."""
import ctypes as C

import pytest

FAKE = 0x1000  # a non-null "device pointer" that is never dereferenced: every call below is rejected by a guard first


@pytest.fixture(scope="module")
def L():
    from emoportraits_b200 import lib as L

    if L.DRY_RUN:
        pytest.skip("EMO_DRY_RUN skips the calls")
    L.load()
    return L


def _refused(L, name, desc, match):
    lib = L.load()
    rc = getattr(lib, name)(C.byref(desc), None)
    assert rc == -1, rc                                  # EMO_ERR_INVALID
    msg = lib.emo_last_error().decode()
    assert match in msg, msg


def test_grid_sample3d_guards(L):
    D = L.GridSample3dDesc
    ok = dict(in_=FAKE, in_layout=1, N=1, C=8, Din=4, Hin=4, Win=4, grid=None, theta=FAKE, Dout=4, Hout=4, Wout=4, out=FAKE,
              out_hi=None, out_lo=None, os_n=512, os_c=1, os_d=128, os_h=32, os_w=8, out_lo2=None)

    def desc(**kw):
        return D(**dict(ok, **kw))

    _refused(L, "emo_grid_sample3d", desc(in_=None), "null input")
    _refused(L, "emo_grid_sample3d", desc(grid=FAKE), "exactly one of grid/theta")
    _refused(L, "emo_grid_sample3d", desc(theta=None), "exactly one of grid/theta")
    _refused(L, "emo_grid_sample3d", desc(out=None), "no output")
    _refused(L, "emo_grid_sample3d", desc(N=0), "bad shape")
    _refused(L, "emo_grid_sample3d", desc(Wout=0), "bad shape")
    _refused(L, "emo_grid_sample3d", desc(C=6), "C % 4 == 0 (C=6)")
    _refused(L, "emo_grid_sample3d", desc(in_=FAKE + 4), "16-byte aligned")
    _refused(L, "emo_grid_sample3d", desc(os_w=6), "multiples of 4")


def test_pose_theta_guards(L):
    P = L.PoseDesc
    _refused(L, "emo_pose_theta", P(None, None, 1, 0, 0, FAKE, FAKE, FAKE, None, 0, 0, None, 0.5), "srt or theta_in")
    _refused(L, "emo_pose_theta", P(FAKE, None, 0, 0, 0, FAKE, FAKE, FAKE, None, 0, 0, None, 0.5), "N must be positive")
    _refused(L, "emo_pose_theta", P(FAKE, None, 1, 1, 0, FAKE, FAKE, FAKE, None, 0, 0, None, 0.5), "mix needs source_theta")
    _refused(L, "emo_pose_theta", P(FAKE, None, 1, 0, 0, FAKE, FAKE, FAKE, None, 0, 0, FAKE, 1.5), "smooth_momentum")
    _refused(L, "emo_pose_theta", P(FAKE, None, 1, 0, 0, FAKE, FAKE, FAKE, None, 0, 0, FAKE, 0.5, -0.5), "smooth_one_minus must be in [0,1]")
    # a factor that does not belong to the momentum (zero, the layout before the field, derives it from the momentum)
    _refused(L, "emo_pose_theta", P(FAKE, None, 1, 0, 0, FAKE, FAKE, FAKE, None, 0, 0, FAKE, 0.9, 0.9), "smooth_one_minus must be 1 - smooth_momentum")


def test_mask_processing_guards(L):
    lib = L.load()

    def refused(rc, match):
        assert rc == -1, rc
        assert match in lib.emo_last_error().decode(), lib.emo_last_error().decode()

    refused(lib.emo_parsing_prepare(None, 1, 3, 8, 8, 512, 512, None, None, FAKE, None), "emo_parsing_prepare: bad arguments")
    refused(lib.emo_parsing_prepare(FAKE, 1, 3, 8, 0, 512, 512, None, None, FAKE, None), "emo_parsing_prepare: bad arguments")
    sets = (C.c_uint * 4)(1, 2, 4, 8)
    refused(lib.emo_parsing_masks(FAKE, 1, 33, 8, 8, 8, 8, sets, FAKE, None, None), "1..32 classes")
    refused(lib.emo_parsing_masks(FAKE, 1, 19, 8, 8, 8, 8, None, FAKE, None, None), "emo_parsing_masks: bad arguments")
    refused(lib.emo_resize_area(FAKE, 1, 3, 8, 8, 0, 4, 1.0, 0.0, FAKE, None), "emo_resize_area: bad arguments")
    refused(lib.emo_l2_flush_clean(None, 1 << 20, None), "emo_l2_flush_clean: bad buffer")

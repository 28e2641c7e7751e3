"""CPU tier: the optimiser's argument checks.  xtb_adam_create rejects, before any CUDA call, what its kernels cannot
handle: decreasing segment offsets (two blocks would update the same parameters), an unknown clip mode, a clip
threshold that is not > 0 under a clipping mode, and m / v buffers that float4 accesses would read misaligned.  The
pointers are fake addresses: a rejected call never dereferences them."""
import ctypes as C

import pytest

ALIGNED_M, ALIGNED_V = 0x10000, 0x20000      # fake device addresses, 16-byte aligned


@pytest.fixture(scope="module")
def lib():
    from xingtian_b200 import build, capi
    build.build()
    return capi.lib()


def _create(lib, count=200, clip_mode=2, clip=1.0, seg=(0, 100, 200), m=ALIGNED_M, v=ALIGNED_V):
    arr = (C.c_longlong * len(seg))(*seg)
    h = C.c_void_p()
    rc = lib.xtb_adam_create(count, 1e-3, 0.9, 0.999, 1e-8, clip_mode, clip, arr, len(seg) - 1,
                             C.c_void_p(m), C.c_void_p(v), C.byref(h))
    return rc, h


REJECTED = {
    "decreasing_offsets": (dict(seg=(0, 100, 50, 200)), b"must not decrease"),
    "decreasing_last_pair": (dict(seg=(0, 1, 3, 2, 200)), b"must not decrease"),
    "clip_mode_3": (dict(clip_mode=3), b"unknown clip_mode 3"),
    "clip_mode_negative": (dict(clip_mode=-1), b"unknown clip_mode -1"),
    "global_clip_zero": (dict(clip_mode=1, clip=0.0), b"clip must be > 0"),
    "global_clip_negative": (dict(clip_mode=1, clip=-5.0), b"clip must be > 0"),
    "global_clip_nan": (dict(clip_mode=1, clip=float("nan")), b"clip must be > 0"),
    "per_tensor_clip_zero": (dict(clip_mode=2, clip=0.0), b"clip must be > 0"),
    "per_tensor_clip_negative": (dict(clip_mode=2, clip=-0.5), b"clip must be > 0"),
    "per_tensor_clip_nan": (dict(clip_mode=2, clip=float("nan")), b"clip must be > 0"),
    "m_misaligned_4": (dict(m=ALIGNED_M + 4), b"16-byte aligned"),
    "m_misaligned_8": (dict(m=ALIGNED_M + 8, clip_mode=0), b"16-byte aligned"),
    "v_misaligned_4": (dict(v=ALIGNED_V + 4, clip_mode=1), b"16-byte aligned"),
    "v_misaligned_12": (dict(v=ALIGNED_V + 12), b"16-byte aligned"),
}


@pytest.mark.parametrize("case", list(REJECTED))
def test_adam_create_rejects_before_any_cuda_call(lib, case):
    kw, msg = REJECTED[case]
    launches = lib.xtb_launch_count()
    rc, h = _create(lib, **kw)
    assert rc == -1, (case, rc)                           # XTB_ERR_ARG
    assert not h.value
    assert msg in lib.xtb_last_error(), lib.xtb_last_error()
    assert b"xtb_adam_create" in lib.xtb_last_error()
    assert lib.xtb_launch_count() == launches


@pytest.mark.parametrize("seg", [(0, 100, 150), (5, 100, 200)])
def test_adam_create_rejects_offsets_that_do_not_span_the_bucket(lib, seg):
    launches = lib.xtb_launch_count()
    rc, h = _create(lib, seg=seg)
    assert rc == -1 and not h.value
    assert b"span [0,count]" in lib.xtb_last_error()
    assert lib.xtb_launch_count() == launches

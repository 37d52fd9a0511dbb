"""CPU checks of the handle contract every C-ABI module keeps: a null handle has the error text "null handle" and
destroys as a no-op, a create without an out pointer is SVS_ERR_INVALID, and without a CUDA device a create with valid
arguments is SVS_ERR_NOGPU, leaves *out null, and the Python wrapper raises SvsError."""
import ctypes as C

import numpy as np
import pytest

SVS_ERR_INVALID = -1
SVS_ERR_NOGPU = -5

_i, _p = C.c_int, C.c_void_p
_LEVELS = (C.c_int * 10)(64, 48, 0, 0, 0, 32, 24, 0, 0, 0)   # two svs_match_level {w, h, f, px, py}: w and h are checked
_WORDS = (C.c_float * 64)()
_CAM = (C.c_double * 4)(500.0, 320.0, 240.0, 0.1)
_OPTS = (C.c_int * 8)(-1, 0)   # svs_ba_opts {device, flags, reserved[6]}

# prefix -> (last-error function, create argument types and values before `out`)
HANDLES = {
    "ba": ("svs_last_error", [(_p, C.addressof(_OPTS))]),
    "chol6": ("svs_chol6_last_error", [(_i, -1)]),
    "fast": ("svs_fast_last_error", [(_i, -1), (_i, 640), (_i, 480), (_i, 1000)]),
    "dt": ("svs_dt_last_error", [(_i, -1), (_i, 640), (_i, 480), (_i, 3), (_i, 0)]),
    "dtc": ("svs_dtc_last_error", [(_i, -1), (_i, 640), (_i, 480), (_i, 3)]),
    "prep": ("svs_prep_last_error", [(_i, -1), (_i, 640), (_i, 480), (_i, 3)]),
    "matcher": ("svs_matcher_last_error", [(_i, -1), (_i, 2), (_p, C.addressof(_LEVELS)), (_i, 4), (_i, 128), (_i, 1024)]),
    "pose": ("svs_pose_last_error", [(_i, -1), (_i, 128)]),
    "place": ("svs_place_last_error", [(_i, -1), (_i, 1), (_p, C.addressof(_WORDS)), (_p, C.addressof(_CAM))]),
    "map": ("svs_map_last_error", [(_i, -1)]),
    "constraints": ("svs_constraints_last_error", [(_i, -1)]),
}


def _fn(L, name, restype, *argtypes):
    """`name` with a prototype of its own (the binding's shared CDLL keeps its argtypes)."""
    return C.CFUNCTYPE(restype, *argtypes)(C.cast(getattr(L, name), C.c_void_p).value)


def _create(L, prefix, out):
    args = HANDLES[prefix][1]
    f = _fn(L, f"svs_{prefix}_create", C.c_int, *[t for t, _ in args], C.c_void_p)
    return f(*[v for _, v in args], out)


@pytest.fixture(scope="module")
def lib(svs):
    return svs.lib()


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")


@pytest.mark.parametrize("prefix", sorted(HANDLES))
def test_null_handle(lib, prefix):
    assert _fn(lib, HANDLES[prefix][0], C.c_char_p, C.c_void_p)(None) == b"null handle"
    _fn(lib, f"svs_{prefix}_destroy", None, C.c_void_p)(None)


@pytest.mark.parametrize("prefix", sorted(HANDLES))
def test_create_without_out_is_invalid(lib, prefix):
    assert _create(lib, prefix, None) == SVS_ERR_INVALID


@pytest.mark.parametrize("prefix", sorted(HANDLES))
def test_create_without_gpu(lib, prefix):
    _no_gpu()
    out = C.c_void_p(0x1234)
    assert _create(lib, prefix, C.addressof(out)) == SVS_ERR_NOGPU
    assert not out.value


WRAPPERS = {
    "BundleAdjuster": lambda svs: svs.BundleAdjuster(),
    "BlockCholesky6": lambda svs: svs.BlockCholesky6(),
    "FastGrid": lambda svs: svs.FastGrid(640, 480, 222, 74, 25, 3, 3),
    "DenseTracker": lambda svs: svs.DenseTracker(640, 480),
    "GuidedMatcher": lambda svs: svs.GuidedMatcher([(64, 48, 100.0, 32.0, 24.0), (32, 24, 50.0, 16.0, 12.0)]),
    "FramePreprocessor": lambda svs: svs.FramePreprocessor(640, 480),
    "PoseOptimizer": lambda svs: svs.PoseOptimizer(),
    "DenseTrackerCpuVariant": lambda svs: svs.DenseTrackerCpuVariant(640, 480),
    "ConstraintBuilder": lambda svs: svs.ConstraintBuilder(),
    "DeviceMap": lambda svs: svs.DeviceMap(),
    "PlaceRecognizer": lambda svs: svs.PlaceRecognizer(np.zeros((4, 64), np.float32), (500.0, 320.0, 240.0, 0.1)),
}


@pytest.mark.parametrize("name", sorted(WRAPPERS))
def test_wrapper_without_gpu(svs, name):
    _no_gpu()
    with pytest.raises(svs.SvsError) as e:
        WRAPPERS[name](svs)
    assert e.value.rc == SVS_ERR_NOGPU

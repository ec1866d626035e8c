"""The product's ctypes wrapper (porechop_b200/cpp_function_wrappers.py) bound to the HOST-SIMULATED engine
(tests/sim/_build/libengine_sim.so, see pbsim_cuda.h / build_sim.py) instead of cpp_functions.so.  TESTS ONLY.

The simulated runtime also checks the ordering of the engine's stream operations (pbsim_cuda.h): races() returns the
races found since the last clear_races()."""
import ctypes
import importlib.util
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_sim  # noqa: E402

_cache = {}


def load(flags=None):
    """the wrapper module on the simulated engine; `flags`: extra -D switches of the product sources (a separate library)"""
    key = tuple(flags) if flags else ()
    if key in _cache:
        return _cache[key]
    from porechop_b200 import cpp_function_wrappers as real
    so = build_sim.build(flags=list(flags) if flags else None)
    spec = importlib.util.spec_from_file_location('pb200_sim_wrappers%d' % len(_cache), real.__file__)
    mod = importlib.util.module_from_spec(spec)
    orig = ctypes.CDLL

    def cdll(path, *a, **k):
        return orig(so if os.path.basename(str(path)) == 'cpp_functions.so' else path, *a, **k)
    ctypes.CDLL = cdll
    try:
        spec.loader.exec_module(mod)
    finally:
        ctypes.CDLL = orig
    lib = mod.C_LIB
    lib.pbsim_race_count.restype = ctypes.c_longlong
    lib.pbsim_race_report.restype = ctypes.c_longlong
    lib.pbsim_race_report.argtypes = [ctypes.c_char_p, ctypes.c_longlong]
    lib.pbsim_stream_create.restype = ctypes.c_void_p
    lib.pbsim_device_alloc.restype = ctypes.c_void_p
    lib.pbsim_device_alloc.argtypes = [ctypes.c_longlong]
    lib.pbsim_device_free.argtypes = [ctypes.c_void_p]
    lib.pbsim_upload.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]
    mod.stream_create = lambda: lib.pbsim_stream_create()
    mod.device_alloc = lib.pbsim_device_alloc
    mod.device_free = lib.pbsim_device_free
    mod.upload = lib.pbsim_upload
    mod.races = lambda: _races(lib)
    mod.clear_races = lib.pbsim_race_clear
    _cache[key] = mod
    return mod


def _races(lib):
    """(number of racing access pairs, text report of the distinct races) since the last clear"""
    n = lib.pbsim_race_report(None, 0)
    buf = ctypes.create_string_buffer(int(n) + 1)
    lib.pbsim_race_report(buf, n + 1)
    return int(lib.pbsim_race_count()), buf.value.decode()


def clear_races():
    """wait for the simulated engine's queued work (ignoring a deferred error a test left behind) and forget the races"""
    lib = load().C_LIB
    lib.pb200Synchronize()
    lib.pbsim_race_clear()


def assert_no_races():
    lib = load().C_LIB
    lib.pb200Synchronize()
    n, text = _races(lib)
    assert n == 0, 'stream-ordering check: %d racing accesses\n%s' % (n, text[:6000])

"""TEST INFRASTRUCTURE ONLY.  CPU checkers for the H100 DSP path, built by oracle/Makefile into oracle/_ref/:

  oracle.port  -- ctypes handle on liboracle_port.so, our C restatement (oracle/port/*.c)
  oracle.ref   -- ctypes handle on libsvtav1_ref.so, the UNMODIFIED reference sources compiled in place (C path +
                  intrinsics-only AVX2 files), or None when it has not been built (fresh clone without the reference tree)
  oracle.load(name) -- the cached handle on any library of LIBS, or None when it has not been built

Both handles are loaded at import, building a missing library first: liboracle_port.so always, libsvtav1_ref.so when the
reference tree is present.  The other libraries are only ever built by make(), and loaded by load().

Only tests/, tools/, __graft_entry__ and bench.py's cpu_baseline / --impl reference legs may import this package.  The
product (svt-av1-psy_b200/, libsvtav1_b200.so) never does.
"""
import ctypes as ct
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
# the reference sources the libraries other than liboracle_port.so are compiled from
REFERENCE = os.environ.get("SVT_AV1_REFERENCE", "/root/reference")
LIBS = {
    "port": "liboracle_port.so",
    "ref": "libsvtav1_ref.so",
    "dlf": "libsvtav1_dlf.so",                # deblocking checker (ref_dlf.c)
    "dlf_search": "libsvtav1_dlf_search.so",  # deblocking filter-level search checker (ref_dlf_search.c)
    "pa_stats": "libsvtav1_pa_stats.so",      # picture-analysis statistics checker (ref_pa_stats.c)
    "enc": "libsvtav1_enc.so",                # the whole reference encoder, linked against libsvtav1_b200.so
}
_ON_REF = ("dlf", "dlf_search", "pa_stats")  # take every reference symbol from libsvtav1_ref.so
BUILD_HINT = "build it with `python __graft_entry__.py --oracle` where the reference sources are available"


def reference_present():
    return os.path.isdir(os.path.join(REFERENCE, "Source"))


def _path(name):
    return os.path.join(_HERE, "_ref", LIBS[name])


def make(*targets):
    """oracle/Makefile's targets, on the reference tree at REFERENCE"""
    subprocess.run(["make", "-s", "-j8", "-C", _HERE, "REF=" + REFERENCE, *targets], check=True)


_loaded = {}


def load(name):
    """the ctypes handle on oracle/_ref/LIBS[name], loaded once, or None when it is not built.  libsvtav1_ref.so is
    initialised (ref_glue_init) on loading, and loaded before the checkers that link to it."""
    if name not in _loaded:
        lib = None
        if os.path.exists(_path(name)) and (name not in _ON_REF or load("ref") is not None):
            lib = ct.CDLL(_path(name))
            if name == "ref":
                lib.ref_glue_init.restype = None
                lib.ref_glue_init()
        _loaded[name] = lib
    return _loaded[name]


if not os.path.exists(_path("port")):
    make("port")
if not os.path.exists(_path("ref")) and reference_present():
    make("ref")
port = load("port")
ref = load("ref")


def p(a, byte_off=0):
    """void* to numpy array data (+ byte offset)."""
    if a is None:
        return ct.c_void_p(0)
    return ct.c_void_p(a.ctypes.data + int(byte_off))

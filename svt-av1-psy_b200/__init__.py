"""svt-av1-psy_b200: H100 (sm_90a) tier of SVT-AV1-PSY's inner-loop DSP.

The product is `libsvtav1_b200.so` (hand-written CUDA behind a C ABI, include/svt_b200.h).  This
package is the thin host-side mirror used by tests and bench: it loads the library with ctypes,
verifies that every symbol the header declares is exported, and exposes numpy-level wrappers that
carry the reference's function names (Source/Lib/Codec/aom_dsp_rtcd.h, common_dsp_rtcd.h).

There is no CPU fallback: importing works without a GPU (symbol check only), but any compute call
requires `init()` to have bound an sm_90 device and aborts otherwise.
"""
import ctypes as _ct
import os as _os
import re as _re

_HERE = _os.path.dirname(_os.path.abspath(__file__)) if "__file__" in globals() else None
_PKG_DIR = _os.path.join(_os.path.dirname(_os.path.dirname(_os.path.abspath(__file__))), "svt-av1-psy_b200")
LIB_PATH = _os.path.join(_PKG_DIR, "libsvtav1_b200.so")
HEADER_PATH = _os.path.join(_os.path.dirname(_PKG_DIR), "include", "svt_b200.h")

if not _os.path.exists(LIB_PATH):
    raise ImportError(
        "libsvtav1_b200.so is missing (%s). Run `python __graft_entry__.py` (nvcc, sm_90a) first; "
        "this package has no CPU fallback." % LIB_PATH)

lib = _ct.CDLL(LIB_PATH)


EXPORTS_PATH = _os.path.join(_PKG_DIR, "exports.txt")


def prototypes():
    """The C ABI's functions as [(name, return type, [parameter types])], sorted by name: exports.txt, one prototype
    per line, written from the header when the library is built (__graft_entry__.build_cuda) and committed, so that
    importing needs neither gcc nor the header."""
    with open(EXPORTS_PATH) as f:
        protos = [_re.fullmatch(r"(.+) (svt_b200_\w+)\((.*)\)", x.strip()).groups() for x in f if x.strip()]
    return [(name, ret, params.split(", ") if params else []) for ret, name, params in protos]


def declared_symbols():
    """The C ABI's function names (exports.txt)."""
    return [name for name, _, _ in prototypes()]


def check_exports():
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    if missing:
        raise ImportError("libsvtav1_b200.so does not export: %s" % ", ".join(missing))
    return True


check_exports()

from . import dsp  # noqa: E402
from .dsp import init, shutdown, launch_count  # noqa: E402,F401

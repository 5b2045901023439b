"""TEST INFRASTRUCTURE ONLY.  CPU checkers for the H100 DSP path:

  oracle.port  -- ctypes handle on oracle/_ref/liboracle_port.so, our C restatement (oracle/port/*.c)
  oracle.ref   -- ctypes handle on oracle/_ref/libsvtav1_ref.so, the UNMODIFIED reference sources
                  compiled in place by oracle/Makefile (C path + intrinsics-only AVX2 files), or None
                  when it has not been built (fresh clone without /root/reference).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.  The product (svt-av1-psy_b200/, libsvtav1_b200.so) never does.
"""
import ctypes as ct
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
PORT_PATH = os.path.join(_HERE, "_ref", "liboracle_port.so")
REF_PATH = os.path.join(_HERE, "_ref", "libsvtav1_ref.so")


def _load_port():
    if not os.path.exists(PORT_PATH):
        subprocess.run(["make", "-s", "-C", _HERE, "port"], check=True)
    return ct.CDLL(PORT_PATH)


def _load_ref():
    if not os.path.exists(REF_PATH):
        if os.path.isdir("/root/reference/Source"):
            subprocess.run(["make", "-s", "-j8", "-C", _HERE, "ref"], check=True)
        else:
            return None
    lib = ct.CDLL(REF_PATH)
    lib.ref_glue_init.restype = None
    lib.ref_glue_init()
    return lib


port = _load_port()
ref = _load_ref()


def p(a, byte_off=0):
    """void* to numpy array data (+ byte offset)."""
    if a is None:
        return ct.c_void_p(0)
    return ct.c_void_p(a.ctypes.data + int(byte_off))

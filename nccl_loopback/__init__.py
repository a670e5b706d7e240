"""Build helper of the loopback NCCL stand-in (nccl_loopback/libnccl_loopback.so, SONAME libnccl.so.2).

TEST INFRASTRUCTURE ONLY, like oracle_blocking/: the product package never imports this module.  A process that loads
the stand-in with RTLD_GLOBAL before the library's first NCCL call runs the library's own multi-rank paths (wva_comm_*,
wva_group_* with several devices) with every rank on one GPU; see nccl_loopback.cpp for what it does and
tests/nccl_loopback_driver.py for the process that uses it.
"""
import os
import subprocess

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "libnccl_loopback.so")
SOURCES = [os.path.join(_DIR, f) for f in ("nccl_loopback.cpp", "exports.map", "Makefile")]


def build(force=False):
    """Build the stand-in (force: even when it is newer than its sources); returns its path."""
    if (not force and os.path.exists(LIB_PATH)
            and os.path.getmtime(LIB_PATH) >= max(os.path.getmtime(s) for s in SOURCES)):
        return LIB_PATH
    subprocess.check_call(["make", "-C", _DIR, "-B", "libnccl_loopback.so"], stdout=subprocess.DEVNULL)
    return LIB_PATH

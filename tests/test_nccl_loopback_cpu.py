"""CPU: the loopback NCCL stand-in (nccl_loopback/) builds, binds where the library looks for NCCL, and offers exactly
the entry points the library resolves; the torch-free driver of tests/test_nccl_loopback_gpu.py gets the stand-in's
unique id through the library and refuses to run beside another libnccl; the packed chunk of the limited solve's
all-gather holds every rank's rows on every plan the GPU tests run."""
import os
import re
import shutil
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rank_emulation as re_  # noqa: E402
from test_nccl_loopback_gpu import COMM_CASES, DRIVER, GROUP_CASES, chunk_bytes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def stand_in():
    import nccl_loopback
    return nccl_loopback.build()


def test_soname(stand_in):
    out = subprocess.check_output(["readelf", "-d", stand_in]).decode()
    assert re.search(r"\(SONAME\)\s+Library soname: \[libnccl\.so\.2\]", out), out


def test_exports_are_what_the_library_resolves(wva, stand_in):
    from inferno_autoscaler_b200 import binding
    out = subprocess.check_output(["nm", "-D", "--defined-only", stand_in]).decode().split()
    exported = {w for w in out if w.startswith("nccl")}
    with open(binding.LIB_PATH, "rb") as f:
        wanted = {m.decode() for m in re.findall(rb"(nccl[A-Z][A-Za-z]{3,})\x00", f.read())}
    assert exported == wanted and len(wanted) == 8, (exported, wanted)
    assert "loopback_counters" in out


def run_driver(tmp_path, prefix=()):
    dst = str(tmp_path / "out.npz")
    cmd = [sys.executable] + list(prefix) + [DRIVER, "unique_id", str(tmp_path / "none.npz"), dst]
    return subprocess.run(cmd, capture_output=True, timeout=300), dst


def test_unique_id_through_the_library(stand_in, tmp_path):
    import numpy as np
    p, dst = run_driver(tmp_path)
    assert p.returncode == 0, p.stderr.decode()
    uid = bytes(np.load(dst)["id"])
    assert len(uid) == 128 and uid.startswith(b"nccl-loopback:")


def test_driver_refuses_another_libnccl(stand_in, tmp_path):
    other = tmp_path / "elsewhere" / "libnccl.so.2"
    other.parent.mkdir()
    shutil.copy(stand_in, other)
    pre = "import ctypes, runpy, sys; ctypes.CDLL(%r); sys.argv = sys.argv[1:]; runpy.run_path(sys.argv[0], run_name='__main__')"
    p, dst = run_driver(tmp_path, prefix=("-c", pre % str(other)))
    assert p.returncode == 3, (p.returncode, p.stderr.decode())
    assert b"libnccl mapped besides the stand-in" in p.stderr and not os.path.exists(dst)


@pytest.mark.parametrize("name,G", sorted(set(COMM_CASES) | {(n, g) for n, g in GROUP_CASES if n != "W"}))
def test_chunk_holds_every_shard(name, G):
    img = re_._image(name)
    S, A = img.S, img.A
    n = chunk_bytes(S, A, G)
    assert n % 16 == 0 and n == (16 + -(-S // G) * A * 45 + 15) // 16 * 16
    for f, k in re_.plan(S, G):
        assert k <= -(-S // G) and 16 + k * A * 45 <= n, (f, k)
    assert chunk_bytes(S, A, G) * G >= 16 * G + S * A * 45

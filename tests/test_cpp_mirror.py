"""C++ host mirror (include/b200sa_table.hpp): compiles on CPU; the KATs of
tests/tests.rs run through it on an H100.  The binary goes to pytest's per-test
temporary directory, so the source tree may be read-only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    exe = str(tmp_path / "test_table")
    src = os.path.join(ROOT, "tests", "cpp", "test_table.cpp")
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
           "-L", os.path.join(ROOT, "suffix_b200"), "-lb200sa", "-Wl,-rpath," + os.path.join(ROOT, "suffix_b200")]
    subprocess.check_call(cmd)
    return exe


def test_cpp_mirror_compiles(tmp_path):
    exe = _build(tmp_path)
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_cpp_mirror_kats(tmp_path):
    exe = _build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "cpp mirror ok" in out.stdout, out.stdout + out.stderr

"""How the suite compiles C and C++ against the product: the compilers, the include list of the C++ adapter and
adapter_exe, which builds one of the adapter drivers in tests/cpp.  TEST INFRASTRUCTURE."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "staticmapping_b200")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
CC = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
# the stand-in headers of the reference tree, then the C ABI and the adapter
ADAPTER_INCLUDES = ["-I", os.path.join(ROOT, "tests", "stubs"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(ROOT, "adapter")]
LINK = ["-L", LIBDIR, "-l:libsm_b200.so", "-Wl,-rpath," + LIBDIR]


def adapter_exe(tmp_path, driver, overlay=None):
    """Compiles tests/cpp/<driver>.cc against the adapter and links it with libsm_b200.so -> the executable's path.
    `overlay` names a directory under tests/ searched before tests/stubs, whose headers replace stand-ins there."""
    if CXX is None:
        pytest.skip("no g++")
    exe = str(tmp_path / driver)
    first = ["-I", os.path.join(ROOT, "tests", overlay)] if overlay else []
    r = subprocess.run([CXX, "-std=c++14", "-O1", "-Wall", *first, *ADAPTER_INCLUDES,
                        os.path.join(ROOT, "tests", "cpp", driver + ".cc"), "-o", exe, *LINK],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe

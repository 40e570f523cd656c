"""The C++ adapter for the reference tree must at least parse and type-check against
stand-in headers (the real Eigen/glog/reference headers are absent in this image)."""
import subprocess

import pytest

from cxx import ADAPTER_INCLUDES, CXX


def test_adapter_compiles_against_stubs(tmp_path):
    if CXX is None:
        pytest.skip("no g++")
    src = tmp_path / "t.cc"
    src.write_text('#include "registrators_b200.h"\n'
                   "int main() { static_map::registrator::IcpFastB200* p = nullptr; (void)p;\n  static_map::registrator::NdtB200* q = nullptr; (void)q;\n  static_map::registrator::NdtWithGicpB200* r = nullptr; (void)r;\n  static_map::registrator::IcpUsingPointMatcherB200* u = nullptr; (void)u;\n  static_map::data::InnerCloudType a, b; static_map::registrator::MotionCompensationB200(a, Eigen::Matrix4d(), &b);\n  static_map::registrator::VoxelGridFilterB200(a, 0.1f, &b); return sizeof(*q) + sizeof(*r) > 0 ? 0 : 1; }\n")
    cmd = [CXX, "-std=c++14", "-fsyntax-only", *ADAPTER_INCLUDES, str(src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

"""The C++ VoxelGrid layer (include/mpl_b200/voxel_grid.hpp through the reference's header name
include/compat/planning_ros_utils/voxel_grid.h) compiles without ROS, with the header's own vectors and with Eigen's
(stand-in) types; tests/test_gpu_voxel_grid.py runs the program on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp_path, eigen=False):
    from mpl_ros_b200.build import build_lib
    so = build_lib()
    exe = str(tmp_path / ("test_voxel_grid" + ("_eigen" if eigen else "")))
    flags = ["-DMPL_B200_USE_EIGEN", "-I", os.path.join(ROOT, "oracle", "shim")] if eigen else []
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror"] + flags +
                          ["-I", os.path.join(ROOT, "include", "compat"), "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_voxel_grid.cpp"), "-o", exe, so,
                           "-Wl,-rpath," + os.path.dirname(so)])
    return exe


@pytest.mark.parametrize("eigen", [False, True])
def test_cpp_voxel_grid_compiles_without_ros(tmp_path, eigen):
    assert os.path.exists(build(tmp_path, eigen))

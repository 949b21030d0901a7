"""Runs the solve kernels of csrc/dks_wide.cuh (plans of more than 128 groups) on HOST threads: tests/emu/emu_shim.h maps
the CUDA execution model (threads of a block, __syncthreads, __shared__, warp butterfly sums) onto std::thread +
std::barrier, tests/emu/wide_emu.cpp compiles the very kernel source nvcc compiles and checks link and finish step
against a plain reference, and the float64 product bit for bit against the host's ascending fma chain, at shapes that
hit every tile boundary.  The GPU parity tests of the same path are
tests/test_gpu_wide.py and the configs[3] singleton case of tests/test_gpu_baseline_shapes.py."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def test_wide_solve_kernels_on_host_threads_product_bit_exact(tmp_path):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "wide_emu")
    cmd = [gxx, "-std=c++20", "-O1", "-pthread", "-I" + os.path.join(HERE, "emu"),
           "-I" + os.path.join(REPO, "distributedkernelshap_b200", "csrc"), "-I" + os.path.join(REPO, "include"),
           os.path.join(HERE, "emu", "wide_emu.cpp"), "-o", exe]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, build.stderr
    run = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(run.stdout)
    assert run.returncode == 0, run.stdout + run.stderr
    assert run.stdout.strip().endswith("OK")

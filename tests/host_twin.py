"""The g++ host twin of a dual-compiled kernel source, for the CPU suites.

The routines under trackformer_b200/csrc that nvcc compiles into kernels are compiled here once more by g++, one
"thread" running each CTA (trackformer_b200/csrc/host_device.h), behind the plain C entries of tests/host_build/.
-ffp-contract=off keeps every floating-point operation separately rounded, as the kernels' __f*_rn / __d*_rn are, so
the twin computes the device's values.
"""
import ctypes
import os
import subprocess

HOST_BUILD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_build")
GXX = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared"]


def build(source_name, tmp_dir):
    """Compiles tests/host_build/<source_name>.cpp into a shared library under tmp_dir and loads it."""
    so = os.path.join(str(tmp_dir), f"lib{source_name}.so")
    subprocess.check_call([*GXX, os.path.join(HOST_BUILD, f"{source_name}.cpp"), "-o", so])
    return ctypes.CDLL(so)

"""Packaging: the native core is compiled in-tree for sm_90a (see
mpi4torch_b200/_build.py); ``pip install .`` builds it once at install time.

The reference drives its single C++ TU through ``mpicc``/``mpicxx`` (reference
setup.py:22-58); there is no MPI here, so the stock toolchain (g++ + nvcc)
is all that is needed."""
import os
import sys

from setuptools import find_packages, setup
from setuptools.command.build_py import build_py

ROOT = os.path.dirname(os.path.abspath(__file__))


class BuildWithNative(build_py):
    def run(self):
        sys.path.insert(0, ROOT)
        from mpi4torch_b200 import _build

        _build.build(verbose=True)
        super().run()


setup(
    packages=find_packages(include=["mpi4torch_b200", "mpi4torch_b200.*"]),
    package_data={"mpi4torch_b200": ["csrc/*/*", "_lib/*.so", "_lib/.stamp"]},
    cmdclass={"build_py": BuildWithNative},
)

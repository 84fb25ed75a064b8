"""setup.py -- `pip install -e .` / `python setup.py build_ext --inplace` for ddstore_b200.

Packaging only (the reference's own build is setup.py:18-41: one Cython extension over ddstore.cxx + common.cxx with
mpicc/mpicxx and libfabric). Here the native pieces are built in-tree by __graft_entry__.build(): nvcc
(-gencode arch=compute_90a,code=sm_90a) + g++ -> ddstore_b200/libddstore_b200.so, Cython -> the `pyddstore` module.
"""
import os
import sys

from setuptools import find_packages, setup
from setuptools.command.build_py import build_py

ROOT = os.path.dirname(os.path.abspath(__file__))


class BuildNative(build_py):
    def run(self):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
        super().run()


setup(
    name="ddstore_b200",
    version="0.1.0",
    description="H100-native distributed in-memory sample store with ORNL/DDStore's surface (get() hot path)",
    packages=find_packages(include=["ddstore_b200", "ddstore_b200.*"]),
    package_data={"ddstore_b200": ["libddstore_b200.so", "cython/pyddstore*.so"]},
    cmdclass={"build_py": BuildNative},
    python_requires=">=3.10",
    install_requires=["numpy"],
)

"""Packaging: the native library is compiled for sm_90a at build time when nvcc is present.

Counterpart of ``setup.py`` (which has no native step).
"""
import os
import sys

from setuptools import setup
from setuptools.command.build_py import build_py


class BuildWithNative(build_py):
    def run(self):
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        try:
            from pytensor_federated_b200 import build as native_build

            native_build.build()
        except Exception as ex:  # CPU-only installs still get the gRPC/graph layers
            print(f"warning: native library not built ({ex}); the fused GPU backend will be unavailable")
        super().run()


setup(cmdclass={"build_py": BuildWithNative})

"""Packaging entry: `python setup.py build_ext --inplace` (or `pip install -e .`) compiles every csrc/**/*.cu|cpp for sm_90a into
paddle_b200/_C*.so with the same ninja build `__graft_entry__.build()` uses; `bdist_wheel` ships the prebuilt module.
Parity (role): the reference's setup.py / CMake super-build (L0 of SURVEY.md) - one extension instead of ~60 external deps."""
import os
import sys

from setuptools import Command, setup
from setuptools.command.build_py import build_py

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


class BuildNative(Command):
    description = "compile the sm_90a extension in-tree (nvcc cross-compiles without a GPU)"
    user_options = [("inplace", "i", "ignored: the module is always placed next to the package")]

    def initialize_options(self):
        self.inplace = 1

    def finalize_options(self):
        pass

    def run(self):
        from paddle_b200 import _build

        path = _build.build(verbose=bool(os.environ.get("VERBOSE")))
        print("built", path)


class BuildPy(build_py):
    def run(self):
        if not os.environ.get("PADDLE_B200_SKIP_NATIVE"):
            self.run_command("build_ext")
        super().run()


setup(cmdclass={"build_ext": BuildNative, "build_py": BuildPy})

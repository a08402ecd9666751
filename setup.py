"""Packaging (reference setup.py:24-117): version file, the native extensions, and the packaged configs.

    pip install -e .            # builds the C++ data helpers and the sm_90a CUDA extension in-tree

Both native pieces are compiled by the same code the runtime uses (``libai_b200.data.data_utils.helpers_build`` and
``libai_b200.ops.build``), so an installed tree and a source checkout produce identical binaries.  ``configs/`` is
linked into ``libai_b200/config/configs`` so ``get_config("common/train.py")`` works from an installed package.
"""
import os
import shutil
import subprocess
import sys
from os import path

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py
from setuptools.command.develop import develop

version = "0.1.0"
HERE = path.dirname(path.abspath(__file__))


def write_version_file():
    sha = "unknown"
    try:
        sha = subprocess.check_output(["git", "rev-parse", "HEAD"], cwd=HERE).decode("ascii").strip()
    except Exception:
        pass
    with open(path.join(HERE, "libai_b200", "version.py"), "w") as f:
        f.write(f"__version__ = '{version}'\ngit_version = {sha!r}\n")


def link_configs():
    """``configs/`` → ``libai_b200/config/configs`` (symlink; copy where symlinks are unavailable)."""
    source = path.join(HERE, "configs")
    destination = path.join(HERE, "libai_b200", "config", "configs")
    if path.islink(destination):
        os.unlink(destination)
    elif path.isdir(destination):
        shutil.rmtree(destination)
    try:
        os.symlink(os.path.relpath(source, path.dirname(destination)), destination)
    except OSError:
        shutil.copytree(source, destination)


def build_native():
    sys.path.insert(0, HERE)
    from libai_b200.data.data_utils import helpers_build
    from libai_b200.ops import build as ops_build

    helpers_build.ensure_built()
    ops_build.build()          # nvcc -gencode arch=compute_90a,code=sm_90a (cross-compiles without a GPU)


class BuildNative(Command):
    description = "compile the C++ data helpers and the sm_90a CUDA extension in-tree"
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        build_native()


class BuildPy(build_py):
    def run(self):
        build_native()
        super().run()


class Develop(develop):
    def run(self):
        build_native()
        super().run()


if __name__ == "__main__":
    write_version_file()
    link_configs()
    setup(
        name="libai_b200",
        version=version,
        description="Hopper-native toolbox for large-scale distributed parallel training",
        packages=find_packages(exclude=("tests", "tests.*", "projects", "projects.*")),
        package_data={"libai_b200": ["*.so", "csrc/*", "data/data_utils/*.so", "data/data_utils/*.cpp",
                                     "config/configs/**/*.py"]},
        python_requires=">=3.9",
        install_requires=["torch>=2.6", "numpy", "pyyaml", "tqdm", "regex", "sentencepiece", "cloudpickle", "tabulate",
                          "termcolor", "safetensors"],
        cmdclass={"build_native": BuildNative, "build_py": BuildPy, "develop": Develop},
    )

"""Packaging: builds the sm_90a extension in-tree, then installs the python package."""
import os
import subprocess
import sys

from setuptools import find_packages, setup
from setuptools.command.build_py import build_py

HERE = os.path.dirname(os.path.abspath(__file__))


class BuildWithKernels(build_py):

  def run(self):
    subprocess.check_call([sys.executable, "-m", "distributed_embeddings_b200.ops._build"], cwd=HERE)
    super().run()


setup(
    name="distributed-embeddings-b200",
    version="0.1.0",
    description="H100-native hybrid-parallel embeddings (PyTorch + sm_90a CUDA + NVLink P2P)",
    packages=find_packages(include=["distributed_embeddings_b200", "distributed_embeddings_b200.*"]),
    package_data={"distributed_embeddings_b200": ["_C.so", "ops/csrc/*"]},
    cmdclass={"build_py": BuildWithKernels},
    python_requires=">=3.10",
    install_requires=["torch", "numpy"],
    zip_safe=False,
)

"""``pip install -e . --no-build-isolation`` / ``python setup.py build_ext --inplace``: the native runtime is built IN-TREE by
``adapcc_b200.build`` (nvcc -gencode arch=compute_90a,code=sm_90a → ``adapcc_b200/_C/libadapcc.so``, loaded with ctypes), so
the packaging step only has to call it. The reference has no packaging at all (a Makefile producing ``communicator.so`` in the
source directory, /root/reference/Makefile:3-19)."""
import os
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


class build_native(Command):
    description = "compile adapcc_b200/csrc for sm_90a into adapcc_b200/_C/libadapcc.so"
    user_options = [("force", "f", "rebuild even if the sources did not change"), ("inplace", "i", "accepted for compatibility")]
    boolean_options = ["force", "inplace"]

    def initialize_options(self):
        self.force = False
        self.inplace = True

    def finalize_options(self):
        pass

    def run(self):
        from adapcc_b200.build import build

        print("native runtime:", build(force=bool(self.force)))


class build_py_with_native(build_py):
    def run(self):
        self.run_command("build_ext")
        super().run()


setup(
    name="adapcc_b200",
    version="0.2.0",
    description="Adaptive collective communication for distributed training, native to H100 over NVLink / NVSwitch",
    packages=find_packages(include=["adapcc_b200", "adapcc_b200.*"]),
    package_data={"adapcc_b200": ["_C/libadapcc.so", "_C/check_p2p", "csrc/*", "csrc/bin/*"]},
    python_requires=">=3.10",
    install_requires=[],                      # torch, numpy, scipy, grpcio are expected in the environment (no index here)
    cmdclass={"build_ext": build_native, "build_py": build_py_with_native},
)

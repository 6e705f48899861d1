"""Packaging for ring_attention_pytorch_b200 (counterpart of the reference's setup.py:1-31).

``pip install -e .`` / ``python setup.py build_ext --inplace`` compile ``csrc/`` for sm_90a with the in-tree
builder (``ring_attention_pytorch_b200/build.py``: nvcc per .cu, g++ for the runtime, one ``_C.so`` next to the
package) — the same artefact ``__graft_entry__.build()`` and the test-suite use, so there is exactly one build path.
"""
from pathlib import Path

from setuptools import Command, find_packages, setup
from setuptools.command.build_ext import build_ext as _build_ext
from setuptools.command.build_py import build_py as _build_py

ROOT = Path(__file__).resolve().parent


def _compile_native():
    import importlib.util

    spec = importlib.util.spec_from_file_location("rab_build", ROOT / "ring_attention_pytorch_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()


class build_ext(_build_ext):
    def run(self):
        _compile_native()


class build_py(_build_py):
    def run(self):
        _compile_native()
        super().run()


class build_native(Command):
    description = "compile the sm_90a extension in-tree"
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        _compile_native()


setup(
    name="ring-attention-pytorch-b200",
    version="0.1.0",
    description="Hopper-native (sm_90a wgmma/TMA + NVLink) ring attention, striped / zig-zag context "
                "parallelism and tree-attention decoding",
    packages=find_packages(include=["ring_attention_pytorch_b200", "ring_attention_pytorch_b200.*"]),
    package_data={"ring_attention_pytorch_b200": ["_C.so", "csrc/*"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.6", "beartype"],  # beartype is optional at run time (utils/validate.py)
    extras_require={"test": ["pytest", "hypothesis", "click"]},
    cmdclass={"build_ext": build_ext, "build_py": build_py, "build_native": build_native},
    zip_safe=False,
)

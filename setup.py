"""Packaging of neuronx_distributed_b200.

    pip install -e .            development install: the CUDA extension is compiled in-tree on first use (or by `build_ext`)
    python setup.py build_ext   compile the sm_90a extension now (nvcc cross-compiles without a GPU)
    pip wheel .                 wheel with the prebuilt extension inside the package (platform wheel, sm_90a only)

Console scripts mirror the reference's (`nxd_convert_zero_checkpoints`, reference setup.py:62-64) and add the sharded-checkpoint
converter that the reference ships as a plain script (`scripts/checkpoint_converter.py`)."""
import os

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py
from setuptools.dist import Distribution

ROOT = os.path.dirname(os.path.abspath(__file__))
version = {}
exec(open(os.path.join(ROOT, "neuronx_distributed_b200", "_version.py")).read(), version)


class BinaryDistribution(Distribution):
    def has_ext_modules(self):                   # platform wheel: it carries a CUDA shared object
        return True


class build_ext(Command):
    """Compile csrc/*.cu + csrc/*.cpp into neuronx_distributed_b200/_build/ (same entry point as `__graft_entry__.build()`)."""
    description = "compile the sm_90a CUDA extension in-tree"
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        import sys

        sys.path.insert(0, ROOT)
        from neuronx_distributed_b200.ops import build as ext_build

        print("built", ext_build.build(verbose=False))


class build_py_with_extension(build_py):
    def run(self):
        if os.environ.get("NXD_SKIP_EXT_BUILD", "0") != "1":
            self.run_command("build_ext")
        super().run()


setup(
    name="neuronx-distributed-b200",
    version=version["__version__"],
    description="Tensor / pipeline / sequence / context / expert parallel training and inference for NVIDIA H100 (sm_90a): "
                "PyTorch + hand-written wgmma / TMA kernels + NCCL / NVSwitch",
    packages=find_packages(include=["neuronx_distributed_b200", "neuronx_distributed_b200.*"]),
    package_data={"neuronx_distributed_b200": ["_build/*.so"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.4", "numpy", "safetensors"],
    extras_require={"test": ["pytest", "pytest-timeout"], "hf": ["transformers"], "s3": ["boto3"]},
    entry_points={"console_scripts": [
        "nxd_convert_zero_checkpoints=neuronx_distributed_b200.optimizer.convert_zero_checkpoints:main",
        "nxd_checkpoint_converter=neuronx_distributed_b200.scripts.checkpoint_converter:main",
    ]},
    distclass=BinaryDistribution,
    cmdclass={"build_ext": build_ext, "build_py": build_py_with_extension},
)

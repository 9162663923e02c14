"""Packaging for unicore-b200.

``pip install -e .`` installs the pure-Python framework (``unicore``, ``unicore_cli``,
``unicore_b200``) and the ``unicore-train`` console script.  The sm_90a extension
``unicore_b200._C`` is built in-tree with ``python setup.py build_ext --inplace`` (needs nvcc;
skipped automatically when nvcc is absent or ``UNICORE_NO_CUDA_EXT=1``).  Unlike the reference
(eight opt-in extensions targeting sm_70/80/90, ``setup.py:141-387``) there is ONE extension and it
targets ``-gencode arch=compute_90a,code=sm_90a`` only.
"""
import os
import shutil

from setuptools import find_packages, setup

ext_modules = []
cmdclass = {}
if shutil.which("nvcc") and os.environ.get("UNICORE_NO_CUDA_EXT", "0") != "1":
    try:
        from unicore_b200.utils.build import cuda_extension, build_ext_class

        ext_modules = [cuda_extension()]
        cmdclass = {"build_ext": build_ext_class()}
    except Exception as exc:  # noqa: BLE001
        print("CUDA extension disabled:", exc)

setup(
    name="unicore-b200",
    version="0.1.0",
    description="Hopper-native (H100) distributed training framework with the Uni-Core API",
    packages=find_packages(exclude=["tests", "tests.*", "baseline", "bench", "profiles"]),
    include_package_data=True,
    python_requires=">=3.9",
    install_requires=["numpy", "torch>=2.4"],
    extras_require={"data": ["lmdb", "tokenizers"], "logging": ["tensorboardX", "wandb"]},
    entry_points={"console_scripts": ["unicore-train = unicore_cli.train:cli_main"]},
    ext_modules=ext_modules,
    cmdclass=cmdclass,
)

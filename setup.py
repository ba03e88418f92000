"""Packaging for tensorflowonspark_b200 (counterpart of the reference's setup.py / setup.cfg).

The CUDA extension is NOT built through setuptools' build_ext: it is compiled in-tree for sm_90a
by ``tensorflowonspark_b200/_build.py`` (``python -c "import __graft_entry__ as g; g.build()"`` or
``scripts/build_ext.sh``) so that the resulting ``_ext/_tfos_b200_C.so`` sits next to the sources
and travels with a checkout; ``pip install -e .`` then only registers the packages.
"""
from setuptools import find_packages, setup

setup(
    name="tensorflowonspark-b200",
    version="0.2.0",
    description="Hopper-native (sm_90a) framework with the capabilities of TensorFlowOnSpark",
    packages=find_packages(include=["tensorflowonspark_b200*", "tensorflowonspark*"]),
    package_data={"tensorflowonspark_b200": ["_ext/*.so"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.6", "numpy", "cloudpickle", "msgpack", "pybind11", "ninja"],
    extras_require={"spark": ["pyspark>=3.1"], "remote_fs": ["pyarrow"], "metrics": ["prometheus_client"],
                    "test": ["pytest", "pytest-timeout", "hypothesis", "protobuf"]},
    entry_points={"console_scripts": [
        "tfos-b200-inference=tensorflowonspark_b200.inference:main",
        "tfos-b200=tensorflowonspark_b200.__main__:main",
    ]},
)

"""pip install -e . builds the native module in-tree (tools/build_native.py) and installs the
`infinistore` console script (reference counterpart: setup.py:31-74, which runs `make`)."""
import os
import sys

from setuptools import Distribution, find_packages, setup
from setuptools.command.build_py import build_py
from setuptools.command.develop import develop

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def get_version() -> str:
    """`<latest tag>.<commits since>` as the reference does (setup.py:7-28); without a tag
    (this repository has none yet) 0.2.0.dev<commit count>, and 0.2.0 outside a checkout."""
    import subprocess

    def git(*a):
        return subprocess.check_output(["git", *a], cwd=ROOT, stderr=subprocess.DEVNULL).decode().strip()

    try:
        try:
            tag = git("describe", "--tags", "--abbrev=0")
            return f"{tag.lstrip('v')}.{git('rev-list', f'{tag}..HEAD', '--count')}"
        except subprocess.CalledProcessError:
            return f"0.2.0.dev{git('rev-list', 'HEAD', '--count')}"
    except Exception:  # noqa: BLE001 - sdist / no git
        return "0.2.0"


def _build_native():
    from tools import build_native

    build_native.build()


class BuildPy(build_py):
    def run(self):
        _build_native()
        super().run()


class Develop(develop):
    def run(self):
        _build_native()
        super().run()


class BinaryDistribution(Distribution):
    """The package ships a prebuilt CPython extension: tag the wheel for this platform/ABI."""

    def has_ext_modules(self):
        return True


setup(
    distclass=BinaryDistribution,
    name="infinistore-b200",
    version=get_version(),
    description="H100-native KV-cache block store with infiniStore's API",
    packages=find_packages(include=["infinistore_b200", "infinistore_b200.*", "infinistore"]),
    package_data={"infinistore_b200": ["_infinistore*.so"]},
    python_requires=">=3.10",
    install_requires=["torch", "numpy", "fastapi", "uvicorn"],
    entry_points={"console_scripts": ["infinistore=infinistore_b200.server:main"]},
    cmdclass={"build_py": BuildPy, "develop": Develop},
)

"""Editable install is optional: tests/bench add the repo root to sys.path themselves.
`python setup.py build_ext --inplace` (or `python -m colossalai_b200.kernel.build`) compiles every native library
for sm_90a into colossalai_b200/kernel/_build/."""
from setuptools import find_packages, setup
from setuptools.command.build_ext import build_ext as _build_ext


class build_ext(_build_ext):
    def run(self):
        import sys, os
        sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
        from colossalai_b200.kernel.loader import build_all

        for p in build_all(verbose=False):
            print("built", p)


setup(
    name="colossalai_b200",
    version="0.1.0",
    packages=find_packages(include=["colossalai_b200", "colossalai_b200.*"]),
    package_data={"colossalai_b200.kernel": ["csrc/*", "_build/*.so"]},
    cmdclass={"build_ext": build_ext},
    entry_points={"console_scripts": ["colossalai_b200=colossalai_b200.cli:cli"]},
    python_requires=">=3.10",
)

"""Build recipe of the reference package used by the drop-in tests and by bench.py's operator-scope reference leg.

lotus-data/lotus is pure Python: its built form is its installed package directory, `lotus/`. `build()` copies that directory
from a checkout of the reference (LOTUS_REFERENCE, default /root/reference) to oracle/_ref/lotus, a git-ignored build product
that travels with the built tree to machines that have no checkout. Without a checkout it keeps whatever oracle/_ref already
holds. Nothing in the product imports it."""
from __future__ import annotations

import os
import shutil

_HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(_HERE, "_ref")


def source_dir() -> str:
    return os.environ.get("LOTUS_REFERENCE", "/root/reference")


def build() -> str | None:
    """-> the directory that holds `lotus/` (oracle/_ref), or None when neither a checkout nor an earlier build is present."""
    src = os.path.join(source_dir(), "lotus")
    if os.path.isfile(os.path.join(src, "__init__.py")):
        tmp = DST + f".tmp{os.getpid()}"
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(src, os.path.join(tmp, "lotus"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        shutil.rmtree(DST, ignore_errors=True)
        os.replace(tmp, DST)
    return DST if os.path.isfile(os.path.join(DST, "lotus", "__init__.py")) else None

"""Stage the unmodified reference package where the GPU box can import it (test / measurement infrastructure only).

The reference is a RecTools source checkout: the directory named by the RECTOOLS_REFERENCE environment variable, else
the build environment's checkout at /root/reference.  `stage()` -- called by `__graft_entry__.build()` -- copies its
pure-Python package `rectools/` as it lies into the git-ignored `oracle/_ref/` (never into the history), from where it
can travel with the working tree exactly like the built `.so` files.  Without a checkout nothing is staged and the tests
that run the reference package skip.  Together with
`oracle/implicit_stub` (import-only placeholders for the third-party `implicit` package + the oracle's restatement of its
top-k) the UNMODIFIED `rectools.models.*` then run on the GPU box: `rectools_b200.install()` is exercised against the real
`VectorModel` / `ModelBase.recommend` / `DistanceSimilarityModule`, and `bench.py` can time `model.recommend()`.
Nothing on the product path imports from here.
"""
from __future__ import annotations

import os
import shutil
import sys
import typing as tp

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get("RECTOOLS_REFERENCE") or "/root/reference"
DST = os.path.join(HERE, "_ref")
STUB = os.path.join(HERE, "implicit_stub")


def _tree_stamp(root: str) -> tp.Tuple[int, int]:
    n = size = 0
    for base, _dirs, files in os.walk(root):
        for f in files:
            if f.endswith(".py"):
                n += 1
                size += os.path.getsize(os.path.join(base, f))
    return n, size


def stage() -> tp.Optional[str]:
    """Copy `<checkout>/rectools` to `oracle/_ref/rectools` (no-op without the checkout or when up to date)."""
    src = os.path.join(SRC, "rectools")
    if not SRC or not os.path.isdir(src):
        return None
    dst = os.path.join(DST, "rectools")
    if os.path.isdir(dst) and _tree_stamp(dst) == _tree_stamp(src):
        return dst
    shutil.rmtree(dst, ignore_errors=True)
    os.makedirs(DST, exist_ok=True)
    shutil.copytree(src, dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    return dst


def reference_root() -> tp.Optional[str]:
    """Directory to put on sys.path for `import rectools`: the staged copy, else the checkout, else None."""
    for root in (DST, SRC):
        if root and os.path.isfile(os.path.join(root, "rectools", "__init__.py")):
            return root
    return None


def available() -> bool:
    return reference_root() is not None


def add_to_path() -> tp.List[str]:
    """Prepend the reference package and the `implicit` stub to sys.path; returns the entries added."""
    root = reference_root()
    if root is None:
        raise ImportError("the reference package is neither staged (oracle/_ref) nor checked out ($RECTOOLS_REFERENCE or /root/reference)")
    added = []
    for p in (os.path.abspath(STUB), os.path.abspath(root)):
        if p not in sys.path:
            sys.path.insert(0, p)
            added.append(p)
    return added


def remove_from_path(added: tp.Sequence[str]) -> None:
    for p in added:
        if p in sys.path:
            sys.path.remove(p)
    for m in [k for k in sys.modules if k == "rectools" or k.startswith("rectools.") or k == "implicit" or k.startswith("implicit.")]:
        sys.modules.pop(m, None)


if __name__ == "__main__":
    print(stage())

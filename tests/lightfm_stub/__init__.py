"""Puts the `lightfm` stand-in (`tests/lightfm_stub/lightfm`, test infrastructure only) on sys.path in front of the
reference package, so that the unmodified `LightFMWrapperModel` imports.  Used together with
`oracle.stage_reference.add_to_path()`; `remove_from_path` drops the stub, every `rectools` module and the stub's module
again, so that later tests import the reference package as they would without it."""
from __future__ import annotations

import os
import sys
import typing as tp

HERE = os.path.dirname(os.path.abspath(__file__))


def add_to_path() -> tp.List[str]:
    """Prepend the stub; drop `rectools` modules imported without it (their optional LightFM import failed)."""
    for m in [k for k in sys.modules if k == "rectools" or k.startswith("rectools.")]:
        sys.modules.pop(m, None)
    if HERE in sys.path:
        return []
    sys.path.insert(0, HERE)
    return [HERE]


def remove_from_path(added: tp.Sequence[str]) -> None:
    for p in added:
        if p in sys.path:
            sys.path.remove(p)
    for m in [k for k in sys.modules if k == "lightfm" or k.startswith("lightfm.") or k == "rectools" or k.startswith("rectools.")]:
        sys.modules.pop(m, None)

"""Drop-in for the reference's ``models`` package (reference lib/models/__init__.py).

Put ``<repo>/litepose_b200/lib`` in front of ``<reference>/lib`` on ``sys.path``:
``models.pose_mobilenet``, ``models.pose_simplenet`` and ``models.pose_supermobilenet`` (what valid.py:130
resolves for MODEL.NAME pose_mobilenet / pose_simplenet / pose_supermobilenet) are the sm_90a-backed modules of this repo;
every other ``models.<name>`` is resolved lazily from the reference tree found further
down ``sys.path`` (out-of-scope model zoo)."""
import importlib
import os
import sys

from . import pose_mobilenet, pose_simplenet, pose_supermobilenet  # noqa: F401

_here = os.path.dirname(os.path.abspath(__file__))
try:
    from .._dynpath import DynPath           # imported as litepose_b200.lib.models
except ImportError:                          # imported as top-level ``models`` (lib/ on sys.path)
    sys.path.insert(0, os.path.dirname(_here))
    try:
        from _dynpath import DynPath
    finally:
        sys.path.pop(0)
__path__ = DynPath(_here, "models")


def __getattr__(name):
    try:
        return importlib.import_module(__name__ + "." + name)
    except ImportError as e:
        raise AttributeError(name) from e

"""make-it-3d_b200: H100-native (sm_90a) implementation of Make-It-3D's SDS training step hot path.

Import with importlib (the directory name contains '-'):  ``mi3d = importlib.import_module("make-it-3d_b200")``
or ``import mi3d_b200`` (alias module at the repo root).
"""
from . import _lib  # noqa: F401
from ._lib import Mi3dError, build, lib  # noqa: F401

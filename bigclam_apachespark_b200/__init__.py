"""bigclam_apachespark_b200 — H100-native drop-in for the F-gradient / line-search step of
thangdnsf/BigCLAM-ApacheSpark (`backtrackingLineSearchs`, codes/bigclam4-7.scala:152-223).

Only what the hot path needs lives here: the CUDA kernels + C ABI (csrc/, libbigclam_b200.so)
and the host-side mirror of the reference's script surface (driver.py).
"""
from ._lib import BigclamError, LIB_PATH, Params  # noqa: F401
from .driver import BigClam, Kset, read_edge_list  # noqa: F401

__all__ = ["BigClam", "Kset", "read_edge_list", "BigclamError", "Params", "LIB_PATH"]

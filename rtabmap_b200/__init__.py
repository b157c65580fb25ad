"""rtabmap_b200 — H100-native loop-closure hot path (detect -> quantise -> score -> verify)
behind the interfaces of rtabmap::VWDictionary / Memory (reference: introlab/rtabmap corelib).

The compute lives in rtabmap_b200/lib/liblcd_b200.so (hand-written sm_90a CUDA behind the C ABI
of include/lcd_b200.h).  This package is the thin Python host side over that ABI; there is no
CPU fallback: importing works anywhere, but creating an engine without a CUDA device raises.
"""
from .capi import LcdError, Engine, load_library, library_path  # noqa: F401
from .vwdictionary import VWDictionaryB200  # noqa: F401

__all__ = ["LcdError", "Engine", "VWDictionaryB200", "load_library", "library_path"]

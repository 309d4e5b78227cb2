"""aigw_b200 — H100-native ext_proc body pipeline (C-ABI library + thin ctypes view).

The product is aigw_b200/libaigw_b200.so (CUDA, sm_90a).  This package only loads it and exposes
the entry points; nothing here computes results on the CPU or touches the test oracle.
"""
from .capi import (AIGW_OK, AIGW_MALFORMED_400, AIGW_INVALID_422, AIGW_INTERNAL, AIGW_DECLINED, SCHEMA, BackendCfg, Context, DocResult, SseResult,
                   load_library, pack_bodies)  # noqa: F401

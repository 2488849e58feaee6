"""serf_b200 — H100-native simulator of serf's SWIM gossip dissemination hot path.

The product is `libserfsim.so` (hand-written sm_90a CUDA kernels behind the C ABI of
include/serfsim.h).  This package is the thin ctypes driver used by the tests and the
bench; it mirrors serf-core's names (MemberStatus, Serf::join/leave/…, Stats).
"""
from .sim import (GossipSim, MemberStatus, MlState, Op, SerfsimError, Config, Stats, TickRow,  # noqa: F401
                  load_library, random_regular_graph, full_mesh_graph, small_world_graph, bind_thread_near_gpu)

__all__ = ["GossipSim", "MemberStatus", "MlState", "Op", "SerfsimError", "Config", "Stats", "TickRow",
           "load_library", "random_regular_graph", "full_mesh_graph", "small_world_graph", "bind_thread_near_gpu"]

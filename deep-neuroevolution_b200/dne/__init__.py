"""dne -- host side of libdne.so: the sm_90a ES/GA rollout-and-update engine.

Only what the hot path needs: the ctypes binding (`_ffi`), network descriptors (`nets`), the device noise slab
(`noise`), the rollout/update engine (`engine`), the batched environment interface (`envs`) and population
sharding (`shard`).  The reference-facing API (same module / function names as the reference) lives in the
sibling package ``es_distributed``.
"""
from . import _ffi  # noqa: F401

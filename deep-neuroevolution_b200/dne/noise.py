"""Device-resident noise slab with the ``SharedNoiseTable`` surface of the reference.

Reference: es_distributed/es.py:51-67 (dup gpu_implementation/neuroevolution/helper.py:27-43):
``noise = RandomState(123).randn(250_000_000)`` cast float64->float32 into fork-shared memory, ``get(i, dim)``
returns the view ``noise[i:i+dim]``, ``sample_index(stream, dim) = stream.randint(0, len(noise)-dim+1)``.

Here the table lives in HBM (1 GB of the 80 GB); every rank holds a full replica.  The values are generated
on the host with numpy's frozen legacy MT19937 / polar Box-Muller stream (bit-identical to the reference) and
uploaded once.  Workers never ship weights or gradients, only (index, return) pairs -- the shared-seed trick of
the reference is kept as is.
"""
from __future__ import annotations

import os

import numpy as np
import torch

NOISE_SEED = 123            # es.py:54
NOISE_COUNT = 250_000_000   # es.py:55
_PAD = 64                   # floats past `count` so aligned 16-byte loads of unaligned slices stay in bounds


def generate_host(count: int = NOISE_COUNT, seed: int = NOISE_SEED, chunk: int = 1 << 24) -> np.ndarray:
    """es.py:60 in chunks (the RandomState stream, including its cached second gaussian, is continuous across
    calls, so chunking does not change the values); avoids the 2 GB float64 transient of the reference."""
    rs = np.random.RandomState(seed)
    out = np.empty(count, dtype=np.float32)
    for s in range(0, count, chunk):
        e = min(count, s + chunk)
        out[s:e] = rs.randn(e - s)
    return out


class SharedNoiseTable:
    """Drop-in for ``es_distributed.es.SharedNoiseTable`` whose storage is a CUDA tensor."""

    def __init__(self, count: int = NOISE_COUNT, seed: int = NOISE_SEED, device=None, host_noise: np.ndarray = None,
                 keep_host: bool = False):
        if not torch.cuda.is_available():
            raise RuntimeError("SharedNoiseTable needs a CUDA device (no CPU fallback)")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        cache = os.environ.get("DNE_NOISE_CACHE")
        if host_noise is None:
            if cache and os.path.exists(cache) and count == NOISE_COUNT and seed == NOISE_SEED:
                host_noise = np.load(cache, mmap_mode="r")
            else:
                host_noise = generate_host(count, seed)
                if cache and count == NOISE_COUNT and seed == NOISE_SEED:
                    try:
                        np.save(cache, host_noise)
                    except OSError:
                        pass
        assert host_noise.dtype == np.float32 and host_noise.ndim == 1
        self.count = int(host_noise.shape[0])
        self._dev = torch.zeros(self.count + _PAD, dtype=torch.float32, device=self.device)
        step = 1 << 26
        for s in range(0, self.count, step):          # staged upload: bounded pinned footprint
            e = min(self.count, s + step)
            self._dev[s:e].copy_(torch.from_numpy(np.ascontiguousarray(host_noise[s:e])))
        self._host = np.asarray(host_noise) if keep_host else None

    def __len__(self):
        return self.count

    @property
    def device_tensor(self) -> torch.Tensor:
        """Full padded slab (bind with ``Context.bind_noise(t, count)``)."""
        return self._dev

    @property
    def noise(self) -> np.ndarray:
        """Host mirror (only if constructed with keep_host=True); the reference exposes ``.noise`` as numpy."""
        if self._host is None:
            raise RuntimeError("no host mirror kept (construct with keep_host=True)")
        return self._host

    def get(self, i: int, dim: int) -> torch.Tensor:
        """es.py:63-64 -- a VIEW of the slab (device tensor)."""
        return self._dev[i:i + dim]

    def sample_index(self, stream: np.random.RandomState, dim: int) -> int:
        """es.py:66-67 -- bit-identical index stream for the same RandomState."""
        return int(stream.randint(0, self.count - dim + 1))

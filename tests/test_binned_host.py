"""Host tests of the discretised-head plumbing: the binned probes of the C ABI (host code, no launch), the bin-table
checks of the environments and the runner, make_runner's choices that need no device, and the head arguments every
driver passes.  No GPU."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dne import _ffi as F                          # noqa: E402
from dne import envs as E                          # noqa: E402
from dne import nets                               # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
DRIVERS = os.path.join(os.path.dirname(HERE), "deep-neuroevolution_b200", "es_distributed")
f32 = np.float32


def _net(ob, hidden, n_out, act=F.ACT_TANH):
    dims = [ob] + list(hidden)
    layers = [nets._dense(dims[i], dims[i + 1], act=act) for i in range(len(hidden))]
    layers.append(nets._dense(dims[-1], n_out, act=F.ACT_NONE))
    return nets._finish(nets.NetSpec("binned", layers, F.OB_VECTOR, ob))


@pytest.mark.parametrize("task,ob,adim", [("pendulum", 3, 1), ("maze", 11, 2)])
def test_binned_probes(task, ob, adim):
    L = F.lib()
    probe = getattr(L, f"dne_{task}_binned_net_supported")
    for nb in (2, 5, 10, 32):
        assert probe(C.byref(_net(ob, (64, 64), adim * nb).desc), nb) == 0, nb
    assert probe(C.byref(_net(ob, (256, 256), adim * 10).desc), 10) == 0          # on a cluster
    assert probe(C.byref(_net(ob, (), adim * 4).desc), 4) == 0                   # the head alone
    for nb, n_out, what in ((1, adim, "2..32 bins"), (33, adim * 33, "2..32 bins"), (0, 0 + adim, "2..32 bins"),
                            (10, adim * 10 + 1, "n_out"), (10, adim * 9, "n_out"), (10, adim, "n_out")):
        assert probe(C.byref(_net(ob, (64, 64), max(n_out, 1)).desc), nb) == -4, (nb, n_out)
        err = L.dne_last_error().decode()
        assert err.startswith(f"dne_{task}_binned_net_supported") and what in err
    assert probe(C.byref(_net(ob, (2048, 2048), adim * 10).desc), 10) == -4
    assert "shared memory" in L.dne_last_error().decode()
    assert probe(C.byref(_net(ob, (64,), adim * 10, act=F.ACT_NONE).desc), 10) == -4   # hidden layers tanh or ReLU
    assert probe(None, 10) == -1
    # the continuous probes still refuse a binned net
    binned = _net(ob, (64, 64), adim * 10)
    assert getattr(L, f"dne_{task}_net_supported")(C.byref(binned.desc)) == -4
    assert getattr(L, f"dne_{task}_cluster_net_supported")(C.byref(binned.desc)) == -4


def test_bin_table_shape_is_checked():
    with pytest.raises(ValueError, match=r"\[2, n_bins\]"):
        E._bin_table(np.zeros((1, 10), f32), 2)
    with pytest.raises(ValueError):
        E._bin_table(np.zeros(10, f32), 1)
    t = E._bin_table(np.arange(10, dtype=np.float64).reshape(2, 5), 2)
    assert t.dtype == f32 and t.flags.c_contiguous and t.shape == (2, 5)


def test_make_runner_without_a_device():
    from dne.rollout import make_runner
    env = E.MazeEnv(2)
    bins = np.zeros((2, 10), f32)
    with pytest.raises(ValueError, match="action_fn"):
        make_runner(None, None, env, action_bins=bins)
    with pytest.raises(NotImplementedError, match="action_bins"):                 # a host map alone is still refused
        make_runner(None, None, env, action_fn=lambda a: a)


class _Fake:
    def __init__(self, bins):
        self._bin_values = bins

    def action_fn(self, scores):
        return scores


def test_runner_head_kw():
    from es_distributed.policies import Policy
    assert Policy.runner_head_kw(_Fake(None)) == {}
    bins = np.zeros((1, 5), f32)
    kw = Policy.runner_head_kw(_Fake(bins))
    assert kw["action_bins"] is bins and kw["action_fn"].__name__ == "action_fn"


@pytest.mark.parametrize("driver", ["es.py", "nses.py", "ga.py", "rs.py", "policies.py"])
def test_every_driver_passes_the_head(driver):
    """Every make_runner call of a driver passes the policy's head arguments (a discretised head dropped here reaches
    the environment as raw scores)."""
    src = open(os.path.join(DRIVERS, driver)).read()
    calls = [c for c in src.split("make_runner(")[1:] if c.startswith(("ctx", "self._ctx"))]
    assert calls, driver
    for c in calls:
        assert "runner_head_kw()" in c[:400], driver

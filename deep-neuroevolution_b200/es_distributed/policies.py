"""``es_distributed.policies`` with the reference's ``Policy`` surface (policies.py:15-113,122-513), backed by libdne.so.

A policy object owns the network descriptor (flat layout = the reference's variable creation order), the flat
parameter vector on the device, observation statistics / the virtual-batch-norm reference batch, and a small slot
engine for ``act``.  Population evaluation does NOT go through per-member ``set_trainable_flat`` calls as in the
reference (es.py:415,419): the drivers hand ``theta`` plus (noise index, scale) per slot to the fused
perturb+forward kernels (dne.rollout.RolloutRunner).
"""
from __future__ import annotations

import logging
import pickle
from typing import Optional

import numpy as np
import torch

from dne import _ffi as F
from dne import nets as N
from dne.engine import SlotForward
from dne.rollout import Unit, make_runner

logger = logging.getLogger(__name__)


def _xavier(rs, shape):
    """contrib.layers default weights_initializer (xavier uniform): limit = sqrt(6/(fan_in+fan_out))."""
    rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
    fan_in, fan_out = shape[-2] * rf, shape[-1] * rf
    lim = np.sqrt(6.0 / (fan_in + fan_out))
    return rs.uniform(-lim, lim, size=shape).astype(np.float32)


def _normc(rs, shape, std):
    """tf_util.py:108-119."""
    out = rs.randn(int(np.prod(shape[:-1])), shape[-1]).astype(np.float32)
    out *= std / np.sqrt(np.square(out).sum(axis=0, keepdims=True))
    return out.reshape(shape)


class Policy:
    """policies.py:15-113."""
    net_name = None

    def __init__(self, *args, **kwargs):
        self.args, self.kwargs = args, kwargs
        self._ctx = kwargs.pop("ctx", None)
        self._seed = kwargs.pop("seed", None)
        self.net: N.NetSpec = self._initialize(*args, **kwargs)
        self.num_params = self.net.num_params
        self.trainable_variables = self._variable_table()
        self.all_variables = list(self.trainable_variables)
        if self._ctx is None:
            from .es import default_context
            self._ctx = default_context()
        self.device = torch.device("cuda", self._ctx.device)
        self._theta = torch.from_numpy(self._initial_theta(np.random.RandomState(self._seed))).to(self.device)
        self._act_engine: Optional[SlotForward] = None
        self.ob_mean = self.ob_std = None
        self.ref_batch: Optional[torch.Tensor] = None
        logger.info('Trainable variables ({} parameters)'.format(self.num_params))
        for name, shp, off in self.trainable_variables:
            logger.info('- {} shape:{} size:{}'.format(name, list(shp), int(np.prod(shp))))

    # -- layout ---------------------------------------------------------------------------------------
    def _variable_table(self):
        """(name, shape, offset) in flat order -- the names the reference's HDF5 snapshots use (policies.py:49-57)."""
        scope = type(self).__name__
        tf_style = self.net.name == "ESAtariPolicy"
        out, bn_i = [], 0
        names = self._layer_names()
        for l, nm in zip(self.net.layers, names):
            wshape = (l.ksize, l.ksize, l.cin, l.cout) if l.kind == F.CONV else (l.cin, l.cout)
            out.append(("{}/{}/{}:0".format(scope, nm, "weights" if tf_style else "w"), wshape, l.off_w))
            if l.off_b >= 0:
                bshape = (l.cout,) if (tf_style or l.kind == F.DENSE) else (1, 1, 1, l.cout)
                out.append(("{}/{}/{}:0".format(scope, nm, "biases" if tf_style else "b"), bshape, l.off_b))
            if l.bn == F.BN_TF:
                bn = "BatchNorm" if bn_i == 0 else "BatchNorm_{}".format(bn_i)
                out.append(("{}/{}/beta:0".format(scope, bn), (l.cout,), l.off_beta))
                out.append(("{}/{}/gamma:0".format(scope, bn), (l.cout,), l.off_gamma))
                bn_i += 1
        return out

    def _layer_names(self):
        raise NotImplementedError

    def _initialize(self, *args, **kwargs):
        raise NotImplementedError

    def _initial_theta(self, rs) -> np.ndarray:
        raise NotImplementedError

    # -- flat get / set (policies.py:102-106; tf_util.py:224-246) --------------------------------------------
    def set_trainable_flat(self, x):
        if isinstance(x, torch.Tensor):
            t = x.to(self.device, torch.float32).reshape(-1)
            # libdne wants a 16-byte aligned base pointer: a row view of a [n, P] matrix (P % 4 != 0) is not
            self._theta = t.clone() if t.data_ptr() % 16 else t
        else:
            x = np.asarray(x, dtype=np.float32)
            assert x.shape == (self.num_params,)
            self._theta = torch.from_numpy(np.ascontiguousarray(x)).to(self.device)

    def get_trainable_flat(self) -> np.ndarray:
        return self._theta.cpu().numpy()

    @property
    def device_theta(self) -> torch.Tensor:
        return self._theta

    def bind_theta(self, t: torch.Tensor):
        """Share the optimizer's device tensor: theta never leaves HBM between generations."""
        self._theta = t

    def reinitialize(self):
        """policies.py:42-44 + tf_util.py:122-130: column-normalise every weight matrix of the CURRENT flat vector to
        its init std and zero the biases (GA: applied to a raw noise slice, ga.py:256-260).  Init-time operation on the
        device tensor (not on the rollout/update hot path; the GA driver uses dne_ga_materialize(mode=1) instead)."""
        self._theta = reinitialize_flat(self.net, self._theta)

    # -- snapshot (policies.py:49-67, 219-249) --------------------------------------------------------------
    # On-disk format = the reference's: one dataset per variable under its TF name + attrs 'name' and
    # 'args_and_kwargs' (pickle).  Container: HDF5 when h5py is importable (reference snapshots load unchanged),
    # else an .npz with the same keys next to the requested name (h5py is not in this image; SURVEY.md 8f rank 2).
    def _all_values(self):
        theta = self.get_trainable_flat()
        vals = {name: theta[off:off + int(np.prod(shp))].reshape(shp) for name, shp, off in self.trainable_variables}
        if self.ob_mean is not None and self.ob_std is not None:        # MujocoPolicy keeps them as variables
            scope = type(self).__name__
            vals["{}/ob_mean:0".format(scope)] = self.ob_mean.cpu().numpy()
            vals["{}/ob_std:0".format(scope)] = self.ob_std.cpu().numpy()
        return vals

    def save(self, filename):
        assert filename.endswith('.h5')
        _write_snapshot(filename, type(self).__name__, pickle.dumps((self.args, dict(self.kwargs)), protocol=-1),
                        self._all_values())

    @classmethod
    def Load(cls, filename, extra_kwargs=None):
        _, blob, data = _read_snapshot(filename)
        args, kwargs = pickle.loads(blob)
        if extra_kwargs:
            kwargs.update(extra_kwargs)
        policy = cls(*args, **kwargs)
        policy.set_all_vars(*[data[name] for name, _, _ in policy.all_variables])
        policy._load_ob_stat(data)
        return policy

    def set_all_vars(self, *vals):
        """policies.py:36-40: assign every variable, in ``all_variables`` order."""
        assert len(vals) == len(self.all_variables), "expected {} arrays".format(len(self.all_variables))
        theta = self.get_trainable_flat()
        for (name, shp, off), v in zip(self.all_variables, vals):
            v = np.asarray(v, dtype=np.float32)
            assert int(v.size) == int(np.prod(shp)), "{}: shape {} != {}".format(name, v.shape, shp)
            theta[off:off + v.size] = v.reshape(-1)
        self.set_trainable_flat(theta)

    def _load_ob_stat(self, data):
        scope = type(self).__name__
        km, ks = "{}/ob_mean:0".format(scope), "{}/ob_std:0".format(scope)
        if km in data and ks in data and np.all(np.isfinite(data[km])) and np.all(np.isfinite(data[ks])):
            self.set_ob_stat(np.asarray(data[km]), np.asarray(data[ks]))

    def initialize_from(self, filename, ob_stat=None):
        """policies.py:219-249: initialise from a snapshot of the SAME architecture (variable names) whose arrays may be
        smaller than this policy's: the loaded values fill the leading sub-array of each variable."""
        _, _, data = _read_snapshot(filename)
        own = {name for name, _, _ in self.all_variables}
        scope = type(self).__name__
        f_names = {k for k in data if not k.endswith(("ob_mean:0", "ob_std:0"))}
        assert own == f_names, 'Variable names do not match'
        theta = self.get_trainable_flat()
        for name, shp, off in self.all_variables:
            f_val = np.asarray(data[name], dtype=np.float32)
            f_shp = f_val.shape
            assert len(shp) == len(f_shp) and all(a >= b for a, b in zip(shp, f_shp)), \
                'This policy must have more weights than the policy to load'
            cur = theta[off:off + int(np.prod(shp))].reshape(shp)
            cur[tuple(np.s_[:n] for n in f_shp)] = f_val
        self.set_trainable_flat(theta)
        km, ks = "{}/ob_mean:0".format(scope), "{}/ob_std:0".format(scope)
        if km in data and ks in data:
            dim = int(self.net.ob_dim)
            init_mean = np.zeros(dim, np.float32)                   # policies.py:236-241: defaults 0 / 0.001
            init_std = np.full(dim, 0.001, np.float32)
            init_mean[:len(data[km])] = data[km]
            init_std[:len(data[ks])] = data[ks]
            if ob_stat is not None:
                ob_stat.set_from_init(init_mean, init_std, init_count=1e5)
            self.set_ob_stat(init_mean, init_std)

    # -- acting ------------------------------------------------------------------------------------------
    def _engine(self, n):
        if self._act_engine is None or self._act_engine.n_slots < n:
            self._act_engine = SlotForward(self._ctx, self.net, max(n, 2))
        return self._act_engine

    def _forward_noiseless(self, ob: np.ndarray):
        n = len(ob)
        eng = self._engine(n)
        eng.set_slots(np.zeros(eng.n_slots, np.int64), np.zeros(eng.n_slots, np.float32),
                      active=(np.arange(eng.n_slots) < n).astype(np.uint8))
        if self.net.needs_ref_batch:
            assert self.ref_batch is not None, "set_ref_batch first (policies.py:332-335)"
            eng.vbn_reference_pass(self._theta, self.ref_batch)
        pad = torch.zeros((eng.n_slots,) + tuple(ob.shape[1:]), dtype=torch.from_numpy(ob[:1]).dtype)
        pad[:n] = torch.from_numpy(np.ascontiguousarray(ob))
        out = eng.forward(self._theta, pad.to(self.device), paired=False, ob_mean=self.ob_mean, ob_std=self.ob_std)
        return out[:n].cpu().numpy()

    def act(self, ob, random_stream=None):
        raise NotImplementedError

    def runner_head_kw(self) -> dict:
        """``make_runner``'s head arguments for this policy: for MujocoPolicy's discretised heads the host map from
        scores to bin values (``action_fn``) and its bin table (``action_bins``, for the episode kernels); nothing for a
        head whose output is the action."""
        bins = getattr(self, "_bin_values", None)
        return {} if bins is None else {"action_fn": self.action_fn, "action_bins": bins}

    def rollout(self, env, *, render=False, timestep_limit=None, save_obs=False, random_stream=None, **_):
        """policies.py:71-97 -- one episode of the CURRENT weights on slot 0 of a ``dne.envs.BatchEnv``.
        Returns (rews_sum_as_array, t, novelty_vector) like the Atari variants (policies.py:429,513)."""
        runner = make_runner(self._ctx, self.net, env, n_slots=2, group=1, pipeline=1, ref_batch=self.ref_batch,
                             **self.runner_head_kw())
        res = runner.run(self._theta, [Unit(0, (0.0,))], timestep_limit, ob_mean=self.ob_mean, ob_std=self.ob_std,
                         collect_bc="final", ac_noise_std=getattr(self, "ac_noise_std", 0.0), random_stream=random_stream)
        return np.array([res.returns[0, 0]], dtype=np.float32), int(res.lengths[0, 0]), res.bcs[0][0]

    @property
    def needs_ob_stat(self):
        raise NotImplementedError

    @property
    def needs_ref_batch(self):
        return self.net.needs_ref_batch

    def set_ob_stat(self, ob_mean, ob_std):
        raise NotImplementedError


class ESAtariPolicy(Policy):
    """policies.py:305-429: conv 16x8x8/4 - BN - relu - conv 32x4x4/2 - BN - relu - fc 256 - BN - relu - out; virtual BN."""

    def _initialize(self, ob_space, ac_space):
        self.ob_space_shape = ob_space.shape
        self.ac_space = ac_space
        self.num_actions = ac_space.n
        return N.make_net("ESAtariPolicy", num_actions=self.num_actions)

    def _layer_names(self):
        return ["conv1", "conv2", "fc", "out"]

    def _initial_theta(self, rs):
        theta = np.zeros(self.net.num_params, dtype=np.float32)
        for l in self.net.layers:
            shp = (l.ksize, l.ksize, l.cin, l.cout) if l.kind == F.CONV else (l.cin, l.cout)
            theta[l.off_w:l.off_w + l.w_size] = _xavier(rs, shp).reshape(-1)
            if l.bn == F.BN_TF:
                theta[l.off_gamma:l.off_gamma + l.cout] = 1.0     # beta 0, gamma 1
        return theta

    def set_ref_batch(self, ref_batch):
        """policies.py:332-335; ref_batch: list/array of 128 observations [84,84,4] (uint8, or float in [0,1])."""
        rb = np.asarray(ref_batch)
        if rb.dtype != np.uint8:
            rb = np.clip(np.rint(rb * 255.0), 0, 255).astype(np.uint8)
        self.ref_batch = torch.from_numpy(np.ascontiguousarray(rb)).to(self.device)
        self.ref_list = [ref_batch, True]

    @property
    def needs_ob_stat(self):
        return False

    def act(self, train_vars, random_stream=None):
        ob = train_vars[0] if isinstance(train_vars, (list, tuple)) else train_vars
        return self._forward_noiseless(np.asarray(ob)).astype(np.int64)


class GAAtariPolicy(Policy):
    """policies.py:433-513: conv 16 - conv 32 - fc 256 - out, normc init, no batch norm."""

    def _initialize(self, ob_space, ac_space, nonlin_type="relu", ac_init_std=0.1):
        self.ob_space_shape = ob_space.shape
        self.ac_space = ac_space
        self.ac_init_std = ac_init_std
        self.num_actions = ac_space.n
        assert nonlin_type == "relu", "only relu is compiled in for the Atari GA policy"
        return N.make_net("GAAtariPolicy", num_actions=self.num_actions, ac_init_std=ac_init_std)

    def _layer_names(self):
        return ["conv1", "conv2", "fc", "out"]

    def _initial_theta(self, rs):
        theta = np.zeros(self.net.num_params, dtype=np.float32)
        for l in self.net.layers:
            shp = (l.ksize, l.ksize, l.cin, l.cout) if l.kind == F.CONV else (l.cin, l.cout)
            theta[l.off_w:l.off_w + l.w_size] = _normc(rs, shp, l.std).reshape(-1)
        return theta

    @property
    def needs_ob_stat(self):
        return False

    def act(self, train_vars, random_stream=None):
        return self._forward_noiseless(np.asarray(train_vars)).astype(np.int64)


class LargeModelPolicy(GAAtariPolicy):
    """The reference GPU path's ``LargeModel`` (gpu_implementation/neuroevolution/models/dqn.py:39-47), P = 4,052,658:
    the "~4M-param conv policy" of the headline configuration."""

    def _initialize(self, ob_space, ac_space, nonlin_type="relu", ac_init_std=0.1):
        self.ob_space_shape = ob_space.shape
        self.ac_space = ac_space
        self.ac_init_std = ac_init_std
        self.num_actions = ac_space.n
        return N.make_net("LargeModel", num_actions=self.num_actions)

    def _layer_names(self):
        return ["conv1", "conv2", "conv3", "fc", "out"]


class SimpleClassifierPolicy(Policy):
    """The reference GPU path's ``SimpleClassifier`` (gpu_implementation/neuroevolution/models/simple.py:29-34): fc1 16 relu,
    fc2 16 relu, linear head over a ``Discrete`` action space, on ``Box`` vector observations (CartPole-v1: P = 386).
    Normc init like ``GAAtariPolicy``; no observation normalisation."""
    model_name = "SimpleClassifier"

    def _initialize(self, ob_space, ac_space):
        assert len(ob_space.shape) == 1, "vector (Box) observations"
        assert hasattr(ac_space, "n"), "a Discrete action space"
        self.ob_space_shape = ob_space.shape
        self.ac_space = ac_space
        self.num_actions = ac_space.n
        return N.make_net(self.model_name, num_actions=self.num_actions, ob_dim=int(ob_space.shape[0]))

    def _layer_names(self):
        return ["fc1", "fc2", "out"]

    def _initial_theta(self, rs):
        theta = np.zeros(self.net.num_params, dtype=np.float32)
        for l in self.net.layers:
            theta[l.off_w:l.off_w + l.w_size] = _normc(rs, (l.cin, l.cout), l.std).reshape(-1)
        return theta

    @property
    def needs_ob_stat(self):
        return False

    def act(self, ob, random_stream=None):
        return np.argmax(self._forward_noiseless(np.asarray(ob, dtype=np.float32)), axis=1).astype(np.int64)


class LinearClassifierPolicy(SimpleClassifierPolicy):
    """The reference GPU path's ``LinearClassifier`` (simple.py:23-27): one linear layer 'out' (CartPole-v1: P = 10)."""
    model_name = "LinearClassifier"

    def _layer_names(self):
        return ["out"]


class MujocoPolicy(Policy):
    """policies.py:122-302 ('ff' connection; 'continuous:', 'uniform:N' and 'custom:v0,..,vk' action heads)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        # Observation statistics from the start: mean 0 / std 1 (the master's initial RunningStat, es.py:26-48) keeps
        # the clip to [-5, 5] on every forward; the engine does not clip inputs fed without statistics.
        dim = int(self.net.ob_dim)
        self.set_ob_stat(np.zeros(dim, np.float32), np.ones(dim, np.float32))

    def _initialize(self, ob_space, ac_space, ac_bins, ac_noise_std, nonlin_type, hidden_dims, connection_type):
        self.ac_space = ac_space
        self.ac_bins = ac_bins
        self.ac_noise_std = ac_noise_std
        self.hidden_dims = hidden_dims
        self.connection_type = connection_type
        assert len(ob_space.shape) == len(ac_space.shape) == 1
        assert connection_type == 'ff'
        mode, arg = ac_bins.split(':')
        adim = ac_space.shape[0]
        low, high = np.asarray(ac_space.low, np.float32), np.asarray(ac_space.high, np.float32)
        self._bin_values = None                       # [adim, num_bins] action value of every bin (discretised heads)
        if mode == 'uniform':                         # policies.py:166-171: bins evenly spaced from low to high
            nb = int(arg)
            self._bin_values = (np.float32(1.0 / (nb - 1.0)) * np.arange(nb, dtype=np.float32)[None, :] * (high - low)[:, None]
                                + low[:, None]).astype(np.float32)
        elif mode == 'custom':                        # policies.py:173-190: listed values in [-1, 1] rescaled to [low, high]
            k = np.array(list(map(float, arg.split(','))), dtype=np.float32)
            assert k.ndim == 1 and k[0] == -1 and k[-1] == 1
            self._bin_values = ((high - low)[:, None] / (k[-1] - k[0]) * (k - k[0])[None, :] + low[:, None]).astype(np.float32)
        elif mode != 'continuous':
            raise NotImplementedError(mode)
        out_dim = adim if self._bin_values is None else adim * self._bin_values.shape[1]   # bins(): dense to dim*num_bins (:116-119)
        return N.make_net("MujocoPolicy", ob_dim=ob_space.shape[0], hidden=tuple(hidden_dims), ac_dim=out_dim,
                          nonlin=nonlin_type)

    def action_fn(self, scores: np.ndarray) -> np.ndarray:
        """Network output -> action.  'continuous:': identity.  Discretised heads (policies.py:116-119,166-190): per action
        dimension the argmax over its bins' scores (first maximum), mapped to that bin's value."""
        if self._bin_values is None:
            return scores
        adim, nb = self._bin_values.shape
        idx = np.argmax(np.asarray(scores).reshape(-1, adim, nb), axis=2)
        return self._bin_values[np.arange(adim)[None, :], idx]

    def _layer_names(self):
        return ["l{}".format(i) for i in range(len(self.hidden_dims))] + ["out"]

    def _initial_theta(self, rs):
        theta = np.zeros(self.net.num_params, dtype=np.float32)
        for l in self.net.layers:
            theta[l.off_w:l.off_w + l.w_size] = _normc(rs, (l.cin, l.cout), l.std).reshape(-1)
        return theta

    def act(self, ob, random_stream=None):
        a = self.action_fn(self._forward_noiseless(np.asarray(ob, dtype=np.float32)))
        if random_stream is not None and self.ac_noise_std != 0:
            a += random_stream.randn(*a.shape) * self.ac_noise_std          # policies.py:204-205
        return a

    @property
    def needs_ob_stat(self):
        return True

    def set_ob_stat(self, ob_mean, ob_std):
        self.ob_mean = torch.from_numpy(np.asarray(ob_mean, dtype=np.float32)).to(self.device)
        self.ob_std = torch.from_numpy(np.asarray(ob_std, dtype=np.float32)).to(self.device)


def reinitialize_flat(net, theta: torch.Tensor) -> torch.Tensor:
    """Column-normalise ``theta`` layer by layer (tf_util.py:122-130 ``normc_initializer`` applied to existing values):
    each weight tensor viewed as [-1, n_out] gets every output column rescaled to L2 norm ``std``; biases -> 0;
    a policy built from slim layers (ESAtariPolicy, policies.py:247-263) has no ``reinitialize`` ops in the reference
    (``v.reinitialize`` raises AttributeError there), and the same error is raised here."""
    if any(l.bn != F.BN_NONE for l in net.layers):
        raise AttributeError("variables of {} carry no reinitialize op (only U.conv / U.dense variables do)".format(net.name))
    out = theta.detach().clone().to(torch.float32).reshape(-1)
    for l in net.layers:
        n_w = (l.ksize * l.ksize * l.cin * l.cout) if l.kind == F.CONV else l.cin * l.cout
        m = out[l.off_w:l.off_w + n_w].view(-1, l.cout)
        m.mul_(float(l.std) / torch.sqrt((m * m).sum(dim=0, keepdim=True)))
        if l.off_b >= 0:
            out[l.off_b:l.off_b + l.cout] = 0
    return out


def _write_snapshot(filename, name, blob: bytes, vals: dict):
    try:
        import h5py
    except ImportError:
        h5py = None
    if h5py is not None:
        with h5py.File(filename, 'w', libver='latest') as f:
            for k, v in vals.items():
                f[k] = v
            f.attrs['name'] = name
            f.attrs['args_and_kwargs'] = np.void(blob)
    else:
        np.savez(filename + ".npz", __name__=name, __args__=np.frombuffer(blob, dtype=np.uint8), **vals)


def _read_snapshot(filename):
    """-> (class name, pickled (args, kwargs), {variable name: array})."""
    import os
    if filename.endswith(".npz") or (not os.path.exists(filename) and os.path.exists(filename + ".npz")):
        data = np.load(filename if filename.endswith(".npz") else filename + ".npz", allow_pickle=False)
        vals = {k: data[k] for k in data.files if not k.startswith("__")}
        return str(data["__name__"]), data["__args__"].tobytes(), vals
    import h5py   # a real HDF5 snapshot (e.g. written by the reference) needs h5py; fail loudly without it
    vals = {}
    with h5py.File(filename, 'r') as f:
        f.visititems(lambda n, obj: vals.__setitem__(n, obj[...]) if isinstance(obj, h5py.Dataset) else None)
        blob = f.attrs['args_and_kwargs'].tobytes()
        name = f.attrs['name']
    return (name.decode() if isinstance(name, bytes) else str(name)), blob, vals

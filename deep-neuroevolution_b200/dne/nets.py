"""Policy network descriptors: the flat parameter layout of each reference policy, as a ``dne_net_desc``.

Flat layout == variable creation order of the reference (SetFromFlat / GetFlat, es_distributed/tf_util.py:224-246;
gpu path gpu_implementation/neuroevolution/models/base.py:165-192):

  LargeModel     models/dqn.py:39-47      conv1[8,8,4,32] b conv2[4,4,32,64] b conv3[3,3,64,64] b fc[7744,512] b out[512,A] b
  Model          models/dqn.py:25-36      conv1[8,8,4,16] b conv2[4,4,16,32] b fc[3872,256] b out[256,A] b
  GAAtariPolicy  policies.py:449-459      same shapes as Model (name/w, name/b)
  ESAtariPolicy  policies.py:319-330      each BN'd layer: weights, biases, BatchNorm/beta, BatchNorm/gamma
  ModelVirtualBN models/batchnorm.py:50-123  Model's layout; layers without bias, 'b' is added AFTER (x-mean)/sqrt(var+eps)
  MujocoPolicy   policies.py:155-162,195  l0..lN dense tanh, 'out' dense (continuous head)
  SimpleClassifier  models/simple.py:29-34  fc1[ob,16] b fc2[16,16] b out[16,A] b (relu hidden; out std 0.1)
  LinearClassifier  models/simple.py:23-27  out[ob,A] b
Kernels are HWIO, activations NHWC, flatten order (h, w, c); conv padding is TF 'SAME'.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

from . import _ffi as F


@dataclass
class LayerSpec:
    kind: int
    cin: int
    cout: int
    ksize: int = 1
    stride: int = 1
    hin: int = 1
    act: int = F.ACT_RELU
    bias: bool = True
    bn: int = F.BN_NONE
    std: float = 1.0            # normc / scale_by std used by the GA initialisers
    off_w: int = 0
    off_b: int = -1
    off_beta: int = -1
    off_gamma: int = -1
    bn_off: int = 0

    @property
    def hout(self) -> int:
        return -(-self.hin // self.stride) if self.kind == F.CONV else 1

    @property
    def pad(self) -> int:
        if self.kind != F.CONV:
            return 0
        total = max((self.hout - 1) * self.stride + self.ksize - self.hin, 0)
        return total // 2

    @property
    def w_size(self) -> int:
        return (self.ksize * self.ksize * self.cin * self.cout) if self.kind == F.CONV else self.cin * self.cout

    @property
    def out_elems(self) -> int:
        return self.hout * self.hout * self.cout if self.kind == F.CONV else self.cout


@dataclass
class NetSpec:
    name: str
    layers: List[LayerSpec]
    ob_kind: int
    ob_dim: int
    num_params: int = 0
    vbn_len: int = 0
    desc: Optional[F.NetDesc] = field(default=None, repr=False)

    @property
    def n_out(self) -> int:
        return self.layers[-1].cout

    @property
    def needs_ref_batch(self) -> bool:
        return self.vbn_len > 0

    def init_std(self) -> List[float]:
        return [l.std for l in self.layers]


def _finish(net: NetSpec) -> NetSpec:
    assert len(net.layers) <= F.DNE_MAX_LAYERS
    off, bn_off = 0, 0
    for l in net.layers:
        l.off_w = off
        off += l.w_size
        if l.bias:
            l.off_b = off
            off += l.cout
        if l.bn == F.BN_TF:                      # contrib.layers creation order: beta, then gamma
            l.off_beta = off
            off += l.cout
            l.off_gamma = off
            off += l.cout
        if l.bn != F.BN_NONE:                    # (mean, var) per channel in the slot's virtual-batch-norm statistics
            l.bn_off = bn_off
            bn_off += 2 * l.cout
    net.num_params = off
    net.vbn_len = bn_off
    d = F.NetDesc()
    d.n_layers = len(net.layers)
    d.ob_kind = net.ob_kind
    d.ob_dim = net.ob_dim
    d.n_out = net.n_out
    d.vbn_len = net.vbn_len
    d.num_params = net.num_params
    for i, l in enumerate(net.layers):
        L = d.layers[i]
        L.kind, L.cin, L.cout, L.ksize, L.stride = l.kind, l.cin, l.cout, l.ksize, l.stride
        L.hin, L.hout, L.pad, L.act, L.bn, L.bn_off = l.hin, l.hout, l.pad, l.act, l.bn, l.bn_off
        L.off_w, L.off_b, L.off_beta, L.off_gamma = l.off_w, l.off_b, l.off_beta, l.off_gamma
    net.desc = d
    return net


def _conv(cin, cout, k, s, hin, **kw):
    return LayerSpec(F.CONV, cin, cout, k, s, hin, **kw)


def _dense(cin, cout, **kw):
    return LayerSpec(F.DENSE, cin, cout, **kw)


def make_net(name: str, num_actions: int = 18, ob_dim: int = 376, hidden: Sequence[int] = (256, 256),
             ac_dim: int = 17, nonlin: str = "tanh", ac_init_std: float = 0.1) -> NetSpec:
    A = num_actions
    if name == "LargeModel":
        layers = [_conv(4, 32, 8, 4, 84), _conv(32, 64, 4, 2, 21), _conv(64, 64, 3, 1, 11),
                  _dense(11 * 11 * 64, 512), _dense(512, A, act=F.ACT_NONE, std=0.1)]
        return _finish(NetSpec(name, layers, F.OB_ATARI_U8, 84 * 84 * 4))
    if name in ("Model", "GAAtariPolicy"):
        layers = [_conv(4, 16, 8, 4, 84), _conv(16, 32, 4, 2, 21),
                  _dense(11 * 11 * 32, 256), _dense(256, A, act=F.ACT_NONE, std=ac_init_std)]
        return _finish(NetSpec(name, layers, F.OB_ATARI_U8, 84 * 84 * 4))
    if name == "ESAtariPolicy":
        layers = [_conv(4, 16, 8, 4, 84, bn=F.BN_TF), _conv(16, 32, 4, 2, 21, bn=F.BN_TF),
                  _dense(11 * 11 * 32, 256, bn=F.BN_TF), _dense(256, A, act=F.ACT_NONE)]
        return _finish(NetSpec(name, layers, F.OB_ATARI_U8, 84 * 84 * 4))
    if name == "ModelVirtualBN":                 # gpu_implementation/neuroevolution/models/batchnorm.py:50-123
        layers = [_conv(4, 16, 8, 4, 84, bn=F.BN_GPU), _conv(16, 32, 4, 2, 21, bn=F.BN_GPU),
                  _dense(11 * 11 * 32, 256, bn=F.BN_GPU), _dense(256, A, act=F.ACT_NONE, std=1.0)]   # 'out': default std (batchnorm.py:106)
        return _finish(NetSpec(name, layers, F.OB_ATARI_U8, 84 * 84 * 4))
    if name == "MujocoPolicy":
        act = {"tanh": F.ACT_TANH, "relu": F.ACT_RELU}[nonlin]
        dims = [ob_dim] + list(hidden)
        layers = [_dense(dims[i], dims[i + 1], act=act) for i in range(len(hidden))]
        layers.append(_dense(dims[-1], ac_dim, act=F.ACT_NONE, std=0.01))
        return _finish(NetSpec(name, layers, F.OB_VECTOR, ob_dim))
    if name == "SimpleClassifier":               # models/simple.py:29-34: fc1 16 relu, fc2 16 relu, out (std 0.1)
        layers = [_dense(ob_dim, 16), _dense(16, 16), _dense(16, A, act=F.ACT_NONE, std=0.1)]
        return _finish(NetSpec(name, layers, F.OB_VECTOR, ob_dim))
    if name == "LinearClassifier":               # models/simple.py:23-27: out only (default std 1.0)
        layers = [_dense(ob_dim, A, act=F.ACT_NONE)]
        return _finish(NetSpec(name, layers, F.OB_VECTOR, ob_dim))
    raise KeyError(f"unknown policy/model type {name!r}")

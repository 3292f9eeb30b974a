"""Generate tests/golden/ref_classifiers.npz by EXECUTING the reference's SimpleClassifier and LinearClassifier.

Run where the reference checkout is available (make_golden_models.REF); nothing under tests/ reads it at test time:
    python tests/golden/make_golden_classifiers.py

gpu_implementation/neuroevolution/models/simple.py builds both classifiers on top of dqn.Model with TensorFlow 1.x calls.
The shape-only TensorFlow stand-in of make_golden_models.py (imported from there, unchanged) is enough to run their
`.make_net()` + `BaseModel.make_weights()` unmodified on a CartPole-shaped input (ob_dim 4, 2 actions) and record

  * the variables in creation order: scoped name, per-member shape, flat offset, `scale_by`;
  * `num_params` (386 and 10).
"""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_models import T, load_reference_models, make_tf   # noqa: E402

OB_DIM, NUM_ACTIONS = 4, 2


def main():
    out = {}
    for cls_name in ("SimpleClassifier", "LinearClassifier"):
        tf = make_tf()
        load_reference_models(tf)
        simple = importlib.import_module("refmodels.simple")
        m = getattr(simple, cls_name)()
        m.make_net(T((1, 1, OB_DIM)), NUM_ACTIONS, batch_size=1)      # Policies x Batch x Features
        m.make_weights()
        names = [v.name for v in m.variables]
        sizes = [int(np.prod(v.shape_[1:])) for v in m.variables]
        out[f"{cls_name}.names"] = np.array(names)
        out[f"{cls_name}.shapes"] = np.array([",".join(map(str, v.shape_[1:])) for v in m.variables])
        out[f"{cls_name}.offsets"] = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        out[f"{cls_name}.sizes"] = np.array(sizes, dtype=np.int64)
        out[f"{cls_name}.var_scale_by"] = np.array([float(v.scale_by) for v in m.variables], dtype=np.float64)
        out[f"{cls_name}.num_params"] = np.int64(m.num_params)
        out[f"{cls_name}.scale_by"] = np.asarray(m.scale_by, dtype=np.float64)
        print(cls_name, "P =", int(m.num_params), "vars:", list(zip(names, sizes)))
    np.savez_compressed(os.path.join(HERE, "ref_classifiers.npz"), **out)
    print("wrote", os.path.join(HERE, "ref_classifiers.npz"))


if __name__ == "__main__":
    main()

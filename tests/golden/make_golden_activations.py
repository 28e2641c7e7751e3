#!/usr/bin/env python
"""Generate activations.npz by EXECUTING the reference's own gelu (xt/model/tf_utils.py:157-166) over
make_golden.TFShim (eager float32), which gains the ops gelu uses: tf.tanh, tf.pow and tf.name_scope.  The function is
taken from the reference file with `ast` and run as written; the other names of that module are not needed.

Recorded:
  x, gelu       a seeded float32 grid (|x| up to 30, dense near 0) and the reference's gelu of it
  act_map_keys  the keys of ACTIVATION_MAP (xt/model/model_utils.py:8-19), read with `ast`, in file order

Needs the reference source tree at make_golden.REF:  python tests/golden/make_golden_activations.py
It writes activations.npz alone; the other fixtures are untouched."""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
from make_golden_gauss import _TFTensor  # noqa: E402


class ActTFShim(mg.TFShim):
    @staticmethod
    def tanh(x):
        return np.tanh(np.asarray(x, np.float32)).astype(np.float32).view(_TFTensor)

    @staticmethod
    def pow(x, y):
        return np.power(np.asarray(x, np.float32), np.float32(y)).astype(np.float32).view(_TFTensor)

    @staticmethod
    def name_scope(name, default_name=None, values=None):
        return mg.TFShim._Ctx()


def _source(relpath):
    with open(os.path.join(mg.REF, relpath)) as f:
        return f.read()


def reference_gelu():
    tree = ast.parse(_source("xt/model/tf_utils.py"))
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "gelu")
    ns = {"tf": ActTFShim, "np": np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "xt/model/tf_utils.py", "exec"), ns)
    return ns["gelu"]


def activation_map_keys():
    tree = ast.parse(_source("xt/model/model_utils.py"))
    for n in tree.body:
        if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "ACTIVATION_MAP" for t in n.targets):
            return [k.value for k in n.value.keys]
    raise RuntimeError("ACTIVATION_MAP not found")


def golden_activations():
    rng = np.random.default_rng(157)
    x = np.concatenate([np.linspace(-30, 30, 601), rng.standard_normal(400) * 3.0, rng.standard_normal(100) * 1e-3,
                        [0.0, 1e-7, -1e-7, 30.0, -30.0]]).astype(np.float32)
    gelu = np.asarray(reference_gelu()(x.view(_TFTensor)), np.float32)
    keys = activation_map_keys()
    np.savez(os.path.join(HERE, "activations.npz"), x=x, gelu=gelu, act_map_keys=np.asarray(keys))
    print("activations.npz", len(x), "points; ACTIVATION_MAP keys", keys)


if __name__ == "__main__":
    if not os.path.isdir(mg.REF):
        sys.exit("needs the reference source tree at %s" % mg.REF)
    golden_activations()

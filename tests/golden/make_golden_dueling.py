#!/usr/bin/env python
"""Generate dueling.npz by EXECUTING the reference's own dueling combine (xt/model/dqn/dqn_mlp.py:80-87):

    layer_normalize(x) = tf.subtract(x, tf.reduce_mean(x, axis=1, keep_dims=True))
    layer_add(x)       = x[0] + x[1]            called as layer_add([adv, layer_normalize(value)])

The two functions are taken from the reference file and run over make_golden.TFShim (eager float32), which gains the
two spellings they use: tf.subtract and TF-1's keep_dims.  Seeded value [B, A] / adv [B, 1] inputs for A in 2, 4, 9, 18.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_dueling.py
It writes dueling.npz alone; the fixtures of make_golden.py are untouched."""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402


class DuelingTFShim(mg.TFShim):
    @staticmethod
    def subtract(a, b): return np.subtract(np.asarray(a, np.float32), np.asarray(b, np.float32))

    @staticmethod
    def reduce_mean(x, axis=None, keepdims=False, keep_dims=None):
        return mg.TFShim.reduce_mean(x, axis=axis, keepdims=keepdims if keep_dims is None else keep_dims)


def reference_functions():
    path = os.path.join(mg.REF, "xt/model/dqn/dqn_mlp.py")
    tree = ast.parse(open(path).read(), path)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("layer_normalize", "layer_add")]
    assert len(keep) == 2
    ns = {"tf": DuelingTFShim()}
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
    return ns["layer_normalize"], ns["layer_add"]


def golden_dueling():
    layer_normalize, layer_add = reference_functions()
    rng = np.random.default_rng(2025)
    out = {}
    for A in (2, 4, 9, 18):
        value = (rng.standard_normal((64, A)) * 3).astype(np.float32)
        adv = rng.standard_normal((64, 1)).astype(np.float32)
        out["value_A%d" % A], out["adv_A%d" % A] = value, adv
        out["q_A%d" % A] = np.asarray(layer_add([adv, layer_normalize(value)]), np.float32)
    np.savez(os.path.join(HERE, "dueling.npz"), **out)


if __name__ == "__main__":
    golden_dueling()

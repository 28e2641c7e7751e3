"""Time DqnInfoFlowModel's device training step (xtb_infoflow_train, targets included) and predict on the GPU, and the
host work of the reference's DQNInfoFlowAlg.train that the step replaces (tiling every next state over its candidates and
the per-transition max loop, with the network itself left out).

The reference ships no config or environment for this model, so every size is an argument and the defaults (vocab
1000, emb_dim 16, user_dim 4, item_dim 2, 100 candidates per transition, a third of the transitions done) are
unverified.  Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def batch(rng, B, a):
    ids = lambda *s: rng.integers(0, a.vocab, s).astype(np.int32)
    cnt = np.full(B, a.candidates)
    return dict(user=ids(B, a.user_dim), click=ids(B, 5 * a.item_dim), noclick=ids(B, 5 * a.item_dim), item=ids(B, a.item_dim),
                next_user=ids(B, a.user_dim), next_click=ids(B, 5 * a.item_dim), next_noclick=ids(B, 5 * a.item_dim),
                cand_off=np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32), cand_item=ids(int(cnt.sum()), a.item_dim),
                reward=rng.uniform(-1, 1, B), done=(rng.random(B) < 1 / 3).astype(np.int32))


def reference_host_ms(b, a, rounds):
    """dqn_infoflw_alg.py:103-153 without the network: np.tile of every next state, the concatenations, and the split /
    argmax loop over Q values."""
    B = len(b["reward"])
    n = np.diff(b["cand_off"])
    q = np.random.default_rng(0).standard_normal(int(n.sum())).astype(np.float32)
    t0 = time.perf_counter()
    for _ in range(rounds):
        nu, nc, nn, ni = [], [], [], []
        for i in range(B):
            k = int(n[i])
            nu.append(np.tile(b["next_user"][i], (k, 1)))
            nc.append(np.tile(b["next_click"][i].reshape(-1, a.item_dim * 5), (k, 1)))
            nn.append(np.tile(b["next_noclick"][i].reshape(-1, a.item_dim * 5), (k, 1)))
            ni.append(b["cand_item"][b["cand_off"][i]:b["cand_off"][i + 1]])
        _ = [np.concatenate(x) for x in (nu, nc, nn, ni)]
        tgt, cur = [], 0
        for i in range(B):
            seg = q[cur:cur + int(n[i])]
            cur += int(n[i])
            tgt.append(b["reward"][i] if b["done"][i] else seg[np.argmax(seg)] * 0.99 + b["reward"][i])
    return (time.perf_counter() - t0) * 1e3 / rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", type=int, default=1000)
    ap.add_argument("--emb-dim", type=int, default=16)
    ap.add_argument("--user-dim", type=int, default=4)
    ap.add_argument("--item-dim", type=int, default=2)
    ap.add_argument("--candidates", type=int, default=100, help="candidate items per transition")
    ap.add_argument("--predict-rows", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("infoflow_step.py needs a CUDA device")
    torch.cuda.set_device(0)
    from xingtian_b200 import capi
    from xingtian_b200.model.dqn_infoflow import DqnInfoFlowModel
    rng = np.random.default_rng(0)
    lib = capi.lib()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "emb.csv")
        np.savetxt(path, rng.standard_normal((a.vocab, a.emb_dim)) * 0.1, delimiter=",")
        m = DqnInfoFlowModel(dict(state_dim=[1], action_dim=1, vocab_size=a.vocab, emb_dim=a.emb_dim, user_dim=a.user_dim,
                                  item_dim=a.item_dim, input_type="int32", embeddings=path, last_activate="linear",
                                  model_config=dict(init_seed=0)))
    m.set_gamma(0.99)
    res = {}
    for B in (32, 256):
        b = batch(rng, B, a)
        for _ in range(a.warmup):
            m._train_packed(b)
        torch.cuda.synchronize()
        l0 = lib.xtb_launch_count()
        t0 = time.perf_counter()
        for _ in range(a.rounds):
            m._train_packed(b)
        torch.cuda.synchronize()
        res["train_ms_b%d" % B] = (time.perf_counter() - t0) * 1e3 / a.rounds
        res["launches_per_step_b%d" % B] = (lib.xtb_launch_count() - l0) // a.rounds
        res["reference_host_ms_b%d" % B] = reference_host_ms(b, a, max(3, a.rounds // 5))
    N = a.predict_rows
    pb = batch(rng, N, a)
    state = dict(user_input=pb["user"], history_click=pb["click"], history_no_click=pb["noclick"], item_input=pb["item"])
    for _ in range(a.warmup):
        m.predict(state)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.rounds * 4):
        m.predict(state)
    res["predict_ms_n%d" % N] = (time.perf_counter() - t0) * 1e3 / (a.rounds * 4)
    name, power = card()
    res.update(gpu=name, power_limit=power, vocab=a.vocab, emb_dim=a.emb_dim, user_dim=a.user_dim, item_dim=a.item_dim,
               candidates=a.candidates)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

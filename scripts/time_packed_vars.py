"""Packed (CSR) against padded [B, L] batches of the variable-name task on one GPU, at the cfg2 and cfg3 model shapes of
bench.py.  Three legs:
  train:   DeviceCorpus.build_vars + ddp_step (ShardedFlatAdam, dropout 0.25) against build_vars_packed + ddp_step;
  predict: Code2Vec.predict on the same batches in both layouts (batches built beforehand);
  host:    c2v_forward_host_async against c2v_forward_host_packed_async from pinned host batches, 4 in flight (the e2e
           leg of bench.py).
Data: the 48 methods of the reference builder's "real" sample (tests/golden/builder_vars.npz) tiled --tiles times, every
tile with its token and path ids remapped at random (without collisions) into the workload's T and P.  That keeps the
sample's distribution of matching contexts per unit; the fill (real contexts / B L) is reported.

First checks that both layouts give the same loss and gradients on units with at least one match (same parameters, same
dropout seed).  Then alternates padded and packed in one process, --rounds times per leg, and reports the median and the
p10-p90 spread of each, with the card name and power limit read in the same run.

    python scripts/time_packed_vars.py [--rounds 20] [--workloads cfg2,cfg3] [--tiles 26] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS  # noqa: E402
from code2vec_b200 import _lib  # noqa: E402
from code2vec_b200 import functional as CF  # noqa: E402
from code2vec_b200.batch_builder import DeviceCorpus  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from time_packed import card, check_same, model, timed  # noqa: E402

DEPTH = 4                                    # host-buffer batches in flight (the session has 4 staging slots)


def corpus(w, tiles, dev, seed=0):
    """the "real" sample tiled `tiles` times, ids remapped per tile into [2, T) (1 is @question) and [1, P)"""
    g = np.load(os.path.join(ROOT, "tests", "golden", "builder_vars.npz"))
    off0, ctx0, units0 = g["real_offsets"], g["real_contexts"].astype(np.int64), g["real_units"]
    rng = np.random.default_rng(seed)
    t_ids = np.unique(np.concatenate([ctx0[:, [0, 2]].ravel(), units0[:, 1]]))
    p_ids = np.unique(ctx0[:, 1])
    n_items = len(off0) - 1
    offs, ctxs, ui, uv = [np.zeros(1, np.int64)], [], [], []
    for k in range(tiles):
        tmap = np.zeros(int(t_ids.max()) + 1, np.int64)
        tmap[t_ids] = 2 + rng.choice(w["T"] - 2, t_ids.size, replace=False)
        pmap = np.zeros(int(p_ids.max()) + 1, np.int64)
        pmap[p_ids] = 1 + rng.choice(w["P"] - 1, p_ids.size, replace=False)
        ctxs.append(np.stack([tmap[ctx0[:, 0]], pmap[ctx0[:, 1]], tmap[ctx0[:, 2]]], 1))
        offs.append(off0[1:] + k * off0[-1])
        ui.append(units0[:, 0] + k * n_items)
        uv.append(tmap[units0[:, 1]])
    c = DeviceCorpus(np.concatenate(offs), np.concatenate(ctxs).astype(np.int32), None, -1, 1, dev)
    n_units = tiles * len(units0)
    c.set_variable_units(np.concatenate(ui), np.concatenate(uv), rng.integers(0, w["C"], n_units), np.zeros(0, np.int64),
                         w["T"])
    return c


def stats(t):
    t = np.asarray(t)
    return float(np.median(t)), float(np.percentile(t, 90) - np.percentile(t, 10))


def alternate(fn, rounds, dev):
    """warm both layouts, then time them alternately -> {padded_ms, packed_ms, speedup, *_spread_ms (p10-p90)}"""
    for layout in ("padded", "packed"):
        for _ in range(3):
            fn(layout)
    t = {"padded": [], "packed": []}
    for _ in range(rounds):
        for layout in ("padded", "packed"):
            t[layout].append(timed(lambda: fn(layout), dev))
    (pm, ps), (km, ks) = stats(t["padded"]), stats(t["packed"])
    return {"padded_ms": pm, "packed_ms": km, "speedup": pm / km, "padded_spread_ms": ps, "packed_spread_ms": ks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--tiles", type=int, default=26, help="copies of the 48-method sample (318 units each)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_packed_vars.py times the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    result = {"card": card(), "rounds": args.rounds, "tiles": args.tiles, "cases": []}
    print(result["card"], flush=True)
    lib = _lib.load()
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    for wname in args.workloads.split(","):
        w = dict(WORKLOADS[wname])
        B, L, H = w["B"], w["L"], w["H"]
        c = corpus(w, args.tiles, dev)
        counts = c.unit_counts
        case = {"workload": wname, "units": int(c.n_units), "B": B, "L": L,
                "fill_corpus": float(np.clip(counts, 1, L).sum() / (c.n_units * L)),
                "units_without_match": int((counts == 0).sum())}
        m = model(w, dev)
        # the two layouts agree: one step on B units with at least one match
        some = np.flatnonzero(counts > 0)[:B]
        s, p, e, lab = c.build_vars(torch.from_numpy(some), L, 1)
        bags, _ = c.build_vars_packed(some, L, 1)
        same = check_same(m, (s, p, e), bags, lab)
        bad = {k: v for k, v in same.items() if v > (1e-5 if k == "loss_rel" else 1e-3)}
        if bad:
            raise SystemExit(f"{wname}: packed and padded differ: {bad}")
        case["same"] = same
        # one epoch's worth of full batches, the same units in both layouts
        order = np.random.default_rng(2).permutation(c.n_units)
        ids = [order[i * B:(i + 1) * B] for i in range(c.n_units // B)]
        dev_ids = [torch.from_numpy(x).to(dev) for x in ids]
        padded = [c.build_vars(d, L, 3) for d in dev_ids]
        packed = [c.build_vars_packed(x, L, 3) for x in ids]
        n_ctx = [bg.N for bg, _ in packed]
        case["fill_batches"] = float(sum(n_ctx) / (len(ids) * B * L))
        print(json.dumps({k: case[k] for k in ("workload", "units", "fill_corpus", "fill_batches")}), flush=True)

        opt = ShardedFlatAdam(m.parameters(), lr=1e-4)      # after the check: it owns the .grad buffers from here on

        def train(layout):
            m.train()
            for i, x in enumerate(ids):
                if layout == "padded":
                    s, p, e, lab = c.build_vars(dev_ids[i], L, 10 + i)
                    ddp_step(m, opt, None, s, p, e, lab, None)
                else:
                    bg, lab = c.build_vars_packed(x, L, 10 + i)
                    ddp_step(m, opt, None, bg, None, None, lab, None)

        def predict(layout):
            m.eval()
            for (s, p, e, _), (bg, _) in zip(padded, packed):
                m.predict(*((s, p, e) if layout == "padded" else (bg, None, None)))

        case["train"] = alternate(train, args.rounds, dev)
        case["predict"] = alternate(predict, args.rounds, dev)
        print(json.dumps({"workload": wname, "train": case["train"], "predict": case["predict"]}), flush=True)
        del opt

        # host-buffer leg: pinned host batches, 4 in flight
        m.eval()
        w_out, b_out = m._head()
        dims = m._dims()
        params = CF.make_params(m.terminal_embedding.weight.data, m.path_embedding.weight.data, m.input_linear.weight.data,
                                m.input_layer_norm.weight.data, m.input_layer_norm.bias.data, m.attention_parameter.data,
                                w_out.data, b_out.data)
        h_pad = [tuple(t.cpu().pin_memory() for t in (s, p, e)) for s, p, e, _ in padded]
        h_pk = [tuple(t.cpu().pin_memory() for t in (bg.starts, bg.paths, bg.ends)) +
                (torch.from_numpy(bg.offsets_host).pin_memory(),) for bg, _ in packed]
        hcv = [torch.empty((B, H)).pin_memory() for _ in range(DEPTH)]
        hat = [torch.empty((B * L,)).pin_memory() for _ in range(DEPTH)]
        hpr = [torch.empty((B,), dtype=torch.int64).pin_memory() for _ in range(DEPTH)]
        hsc = [torch.empty((B,)).pin_memory() for _ in range(DEPTH)]
        sess = ctypes.c_void_p()
        _lib.check(lib.c2v_session_create(0, ctypes.byref(dims), B, L, ctypes.byref(sess)), "session_create")
        tick = ctypes.c_int64(0)
        algo = _lib.ALGO_AUTO | 0x100                         # C2V_FLAG_REUSE_PREP: the weights do not change

        def host(layout):
            pending = []
            for i in range(2 * len(ids)):
                k, j = i % DEPTH, i % len(ids)
                out = (None, P(hcv[k]), P(hat[k]), P(hpr[k]), P(hsc[k]), algo, ctypes.byref(tick))
                if layout == "padded":
                    rc = lib.c2v_forward_host_async(sess, ctypes.byref(params), *(P(t) for t in h_pad[j]), None, B, *out)
                else:
                    rc = lib.c2v_forward_host_packed_async(sess, ctypes.byref(params), *(P(t) for t in h_pk[j]), None, B,
                                                           n_ctx[j], *out)
                _lib.check(rc, layout)
                pending.append(tick.value)
                if len(pending) == DEPTH:
                    _lib.check(lib.c2v_session_wait(sess, pending.pop(0)), "session_wait")
            for t in pending:
                _lib.check(lib.c2v_session_wait(sess, t), "session_wait")

        case["host"] = alternate(host, args.rounds, dev)
        case["host"]["calls_per_round"] = 2 * len(ids)
        case["host"]["h2d_bytes_per_batch"] = {"padded": 24 * B * L,
                                               "packed": float(np.mean([24 * n + 8 * (B + 1) for n in n_ctx]))}
        case["host"]["d2h_attention_bytes_per_batch"] = {"padded": 4 * B * L, "packed": float(np.mean([4 * n for n in n_ctx]))}
        lib.c2v_session_destroy(sess)
        case["train"]["steps_per_round"] = case["predict"]["batches_per_round"] = len(ids)
        print(json.dumps({"workload": wname, "host": case["host"]}), flush=True)
        result["cases"].append(case)
        del m, padded, packed, c
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

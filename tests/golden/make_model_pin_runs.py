"""Record what the reference's model scaffold did in tests/test_reference_model_pin.py's live runs (exported variables fed
to it, restore() of a snapshot written by the package, the train step with prescribed gradients, the per-graph learning
rate, default_params of every model class) into ref_model_pin_runs.pkl.gz:

    TF_GNN_SAMPLES_REFERENCE=<checkout of the original> python tests/golden/make_model_pin_runs.py"""
import gzip
import hashlib
import io
import os
import pickle
import sys
import tempfile
from contextlib import redirect_stdout

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    if p not in sys.path:
        sys.path.insert(0, p)

import batcher_cases as BC                          # noqa: E402
import model_cases as MC                            # noqa: E402
import test_reference_model_pin as P                # noqa: E402

SAMPLE_ROWS, SAMPLE_ELEMS = 48, 64


def digest(a):
    a = np.ascontiguousarray(np.asarray(a, np.float64))
    return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()


def row_sample(n):
    """The fixed sample of rows of a final node-representation matrix that is stored (with the column sums over all rows)."""
    return np.sort(np.random.default_rng(0).permutation(n)[:SAMPLE_ROWS])


def compact(out):
    """Keep the file small: final representations as a fixed row sample + column sums, the restored variables as digests,
    gradients as their first SAMPLE_ELEMS elements + norm (the prescribed ones are regenerated from the hook's call order)."""
    for k, v in out.items():
        if k.startswith("export/"):
            f = v.pop("final")
            v["final_rows"], v["final_sample"], v["final_colsum"] = row_sample(len(f)), f[row_sample(len(f))], f.sum(axis=0)
        elif k.startswith("restore/"):
            v["variables"] = {n: digest(a) for n, a in v["variables"].items()}
        elif k.startswith("train_step/"):
            v["hook_calls"] = [(n, None if g is None else tuple(np.shape(g))) for n, g in v.pop("prescribed").items()]
            v["applied"] = [(None if g is None else (np.ravel(g)[:SAMPLE_ELEMS].copy(), float(np.linalg.norm(g))), n)
                            for g, n in v["applied"]]
    return out


def main():
    out = {}
    import tf1_shim
    from tf1_shim import variables as TV
    with tempfile.TemporaryDirectory() as ppi_dir:
        BC.write_ppi_dir(ppi_dir, "test")
        for name in P.EXPORT_CASES:
            case = MC.CASES[name]
            feed, L = P.repo_feed(case, dict(P.TASK_DEFAULTS[case["task"]], **case["task_params"]), ppi_dir)
            model, _ = P._package_model(case, feed, L, seed=5)
            named = model.to_reference_weights()
            named.pop("total_num_graphs:0")
            provider = TV.provider_from(named)
            r = MC.run_reference(case, np.float64, provider=provider)
            out["export/" + name] = {"final": np.asarray(r["final"], np.float64), "variables": sorted(r["variables"]),
                                     "used": sorted(provider.used), "num_parameters": int(r["num_parameters"]),
                                     "metrics": {k: float(v) for k, v in r["metrics"].items()}}
        for name in P.RESTORE_CASES:
            case = MC.CASES[name]
            task_params = dict(P.TASK_DEFAULTS[case["task"]], out_layer_dropout_keep_prob=1.0, **case["task_params"])
            feed, L = P.repo_feed(case, task_params, ppi_dir)
            model, _ = P._package_model(case, feed, L, seed=9)
            with tempfile.TemporaryDirectory() as d:
                path = os.path.join(d, "snapshot.pickle")
                model.save_reference_snapshot(path, task_params, P.snapshot_metadata(case, task_params, feed, L))
                with tf1_shim.installed(dtype=np.float32) as session:
                    session.feeds = dict(feed, out_layer_dropout_keep_prob=1.0)
                    mu = tf1_shim.import_reference_model_utils()
                    buf = io.StringIO()
                    with redirect_stdout(buf):
                        restored = mu.restore(path, d, run_id="restored")
                    out["restore/" + name] = {"stdout": buf.getvalue().replace(d, "{TMP}"), "model_class": type(restored).__name__,
                                              "num_edge_types": int(restored.task.num_edge_types),
                                              "variables": {k: np.asarray(v) for k, v in session.variables.items()}}
        for optimizer in P.OPTIMIZERS:
            case, hook, prescribed = P.train_step_case(optimizer)
            r = MC.run_reference(case, np.float64, gradient_hook=hook)
            out["train_step/" + optimizer] = {"loss_is_task_loss": bool(r["loss_is_task_loss"]), "optimizers": r["optimizers"],
                                              "params": r["params"], "prescribed": prescribed,
                                              "applied": [(None if g is None else np.asarray(g), n) for g, n in r["applied"]]}
        r = MC.run_reference(P.lr_case(), np.float32)
        out["lr"] = {"optimizers": r["optimizers"], "num_graphs": int(r["feed"]["num_graphs"]), "params": r["params"],
                     "num_edge_types": int(r["num_edge_types"])}
        with tf1_shim.installed():
            tf1_shim.import_reference_task("sparse_graph_task")
            import models
            out["default_params"] = {cls_name: getattr(models, cls_name).default_params() for cls_name in MC.MODEL_CLASSES.values()}
    with gzip.open(os.path.join(HERE, "ref_model_pin_runs.pkl.gz"), "wb") as f:
        pickle.dump(compact(out), f, protocol=4)


if __name__ == "__main__":
    main()

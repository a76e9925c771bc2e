"""Writes tests/golden/ref_model_<case>.npz by running the REFERENCE's own model scaffold and task heads (models/*.py,
tasks/{ppi,qm9}_task.py, unmodified, built eagerly under tests/tf1_shim.graph_mode; see model_cases.py):

    python tests/golden/make_model_fixtures.py [case ...]          (needs the original checkout: TF_GNN_SAMPLES_REFERENCE=<path>)

Per case: the pickle the reference's own save_model wrote (weights under the reference's variable names + params), the
final node representations and task metrics of the float64 run, the float32 run's error against it (err32), and the
"Model has N parameters." count.  The feed is NOT stored: it is the first minibatch of the committed QM9 subset / the seeded
PPI fold, which batching.py reproduces bit-exactly (tests/test_reference_batcher_pin.py)."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import model_cases as MC      # noqa: E402


def make_case(name):
    case = MC.CASES[name]
    r64 = MC.run_reference(case, np.float64)
    r32 = MC.run_reference(case, np.float32)
    assert r32["final"].dtype == np.float32 and r64["final"].dtype == np.float64
    assert all(np.array_equal(r64["variables"][k], r32["variables"][k].astype(np.float64)) for k in r64["variables"])
    scale = float(np.abs(r64["final"]).max())
    blob = {"pickle": np.frombuffer(r64["pickle"], dtype=np.uint8), "final": r64["final"],
            "err32": np.float64(np.abs(r32["final"].astype(np.float64) - r64["final"]).max() / scale),
            "num_parameters": np.int64(r64["num_parameters"]), "num_edge_types": np.int64(r64["num_edge_types"]),
            "num_nodes": np.int64(r64["feed"]["num_nodes"]), "num_graphs": np.int64(r64["feed"]["num_graphs"]),
            "metrics": np.asarray(json.dumps({k: float(v) for k, v in r64["metrics"].items()})),
            "variable_names": np.asarray(sorted(r64["variables"])),
            "meta": np.asarray(json.dumps({"model": r64["model_name"], "task": r64["task_name"],
                                           "source": "reference models/*.py + tasks/*.py via tests/tf1_shim.graph_mode"}))}
    out = os.path.join(HERE, "ref_model_%s.npz" % name)
    np.savez_compressed(out, **blob)
    print("%-34s V=%d params=%d err32=%.2e %.0f KB" % (name, blob["num_nodes"], blob["num_parameters"], blob["err32"],
                                                       os.path.getsize(out) / 1024))


if __name__ == "__main__":
    for n in (sys.argv[1:] or list(MC.CASES)):
        make_case(n)

"""Record what the reference's name factories do (utils/utils.py get_activation / get_aggregation_function / get_gated_unit,
utils/model_utils.py name_to_model_class) and the signatures of its layer functions into ref_utils_outcomes.json:

    TF_GNN_SAMPLES_REFERENCE=<checkout of the original> python tests/golden/make_utils_fixtures.py"""
import inspect
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    if p not in sys.path:
        sys.path.insert(0, p)

import test_reference_utils_pin as U                # noqa: E402
import tf1_shim                                     # noqa: E402


def main():
    out = {"activations": {}, "aggregations": {}, "cells": {}, "models": {}, "signatures": {}}
    x = np.linspace(-3, 3, 25)
    with tf1_shim.installed(dtype=np.float64) as session:
        import utils as ref_utils
        import gnns as ref_gnns
        mu = tf1_shim.import_reference_model_utils()
        tf = session.tf
        for name in U.ACTIVATION_NAMES:
            r = U.outcome(ref_utils.get_activation, name)
            out["activations"][repr(name)] = list(r) if r[0] != "ok" else ["ok", None if r[1] is None else [float(v) for v in r[1](x)]]
        agg_names = {tf.unsorted_segment_sum: "sum", tf.unsorted_segment_max: "max", tf.unsorted_segment_mean: "mean",
                     tf.unsorted_segment_sqrt_n: "sqrt_n"}
        for name in U.AGGREGATION_NAMES:
            r = U.outcome(ref_utils.get_aggregation_function, name)
            out["aggregations"][repr(name)] = list(r) if r[0] != "ok" else ["ok", agg_names[r[1]]]
        for name in U.CELL_NAMES:
            r = U.outcome(ref_utils.get_gated_unit, 8, name, "tanh")
            if r[0] == "ok":
                called = U.outcome(r[1], np.zeros((2, 8)), [np.zeros((2, 8))])
                out["cells"][name] = ["ok", type(r[1]).__name__, called[0]]
            else:
                out["cells"][name] = list(r)
        out["cell_swish"] = list(U.outcome(ref_utils.get_gated_unit, 8, "gru", "swish"))
        for name in U.MODEL_NAMES:
            r = U.outcome(mu.name_to_model_class, name)
            if r[0] != "ok":
                out["models"][name] = list(r)
            else:
                cls, extra = r[1]
                params = cls.default_params()
                params.update(extra)
                out["models"][name] = ["ok", cls.__name__, json.loads(json.dumps(params, default=repr))]
        for n in dir(ref_gnns):
            if n.startswith("sparse_") and n.endswith("_layer"):
                out["signatures"][n] = [[p.name, repr(p.default)] for p in inspect.signature(getattr(ref_gnns, n)).parameters.values()]
    with open(os.path.join(HERE, "ref_utils_outcomes.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()

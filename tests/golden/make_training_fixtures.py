"""Run the reference's epoch loop (tests/test_reference_training_pin.py:run_reference_loop) on the QM9 and PPI set-ups of
that test and record its log lines, feeds and best-model file in ref_training_loops.json, the data directory written as
``{TMP}``:

    TF_GNN_SAMPLES_REFERENCE=<checkout of the original> python tests/golden/make_training_fixtures.py"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    if p not in sys.path:
        sys.path.insert(0, p)

import test_reference_training_pin as T             # noqa: E402


def record(lines, calls, best_file, saved, d):
    return {"lines": [ln.replace(d, "{TMP}") for ln in lines], "best_file": best_file.replace(d, "{TMP}"), "saved": bool(saved),
            "calls": [dict(c, first_feature_row=[float(x) for x in c["first_feature_row"]]) for c in calls]}


def main():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        _, _, test_file = T.write_qm9_data(d)
        out["qm9"] = record(*T.run_reference_loop(data_dir=d, test_path=test_file, **T.QM9_LOOP), d)
    with tempfile.TemporaryDirectory() as d:
        T.write_ppi_data(d)
        out["ppi"] = record(*T.run_reference_loop(data_dir=d, test_path=d, **T.PPI_LOOP), d)
    with open(os.path.join(HERE, "ref_training_loops.json"), "w") as f:
        json.dump(out, f, indent=0)


if __name__ == "__main__":
    main()

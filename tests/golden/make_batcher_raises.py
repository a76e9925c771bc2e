"""Record the exceptions the reference's batchers raise on the inputs of tests/test_reference_batcher_pin.py that it cannot
run (the untied QM9 configurations, a PPI graph without links) into ref_batcher_raises.json:

    TF_GNN_SAMPLES_REFERENCE=<checkout of the original> python tests/golden/make_batcher_raises.py"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    if p not in sys.path:
        sys.path.insert(0, p)

import batcher_cases as BC                          # noqa: E402


def raised(fn, *args):
    try:
        fn(*args)
    except Exception as exc:                        # noqa: BLE001 -- the exception IS the recorded behaviour
        return [type(exc).__name__, str(exc)]
    return None


def main():
    out = {"qm9/" + case: raised(BC.reference_qm9_feeds, *BC.QM9_REFERENCE_RAISES[case]) for case in sorted(BC.QM9_REFERENCE_RAISES)}
    with tempfile.TemporaryDirectory() as d:
        out["ppi/linkless"] = raised(BC.reference_ppi_feeds, {}, 10 ** 6, BC.write_ppi_dir(d, "test", linkless_graph=2))
    with open(os.path.join(HERE, "ref_batcher_raises.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()

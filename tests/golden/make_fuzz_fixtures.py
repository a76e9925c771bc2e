"""Record the reference's outputs for the seeded random cases of tests/test_reference_fuzz.py into ref_fuzz_cases.npz:

    TF_GNN_SAMPLES_REFERENCE=<checkout of the original> python tests/golden/make_fuzz_fixtures.py

Key "<kind>/<i>" holds the reference's float64 output of case i; "<kind>/<i>/exc" the exception type and message it raised."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_ref_fixtures as MRF                     # noqa: E402
import test_reference_fuzz as F                     # noqa: E402


def main():
    out = {}
    for kind in F.KINDS:
        rng = np.random.default_rng(sum(map(ord, kind)))
        for i in range(F.CASES_PER_KIND):
            case, h, adj, indeg, w = F.make_case(kind, rng)
            try:
                ref, _ = MRF.run_reference(case, h, adj, indeg, w, np.float64)
                out["%s/%d" % (kind, i)] = np.asarray(ref, np.float64)
            except Exception as exc:                # noqa: BLE001 -- the exception IS the recorded behaviour
                out["%s/%d/exc" % (kind, i)] = np.array([type(exc).__name__, str(exc)])
    np.savez_compressed(os.path.join(HERE, "ref_fuzz_cases.npz"), **out)


if __name__ == "__main__":
    main()

"""CPU: librgnn reads no environment variable.  The C ABI promises deterministic, bit-reproducible results, so which kernels
run and in what order they sum is chosen from the inputs alone: a process that inherits some variable gets the same
kernels as every other."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tf-gnn-samples_b200", "csrc")


def test_library_sources_never_call_getenv():
    paths = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(ROOT, "include", "rgnn.h")]
    assert any(p.endswith("seg_kernels.cu") for p in paths) and any(p.endswith("layers.cu") for p in paths)
    offenders = []
    for path in paths:
        with open(path, encoding="utf-8") as f:
            for n, line in enumerate(f, 1):
                if "getenv" in line:
                    offenders.append("%s:%d: %s" % (os.path.relpath(path, ROOT), n, line.strip()))
    assert not offenders, "environment-dependent code in librgnn:\n" + "\n".join(offenders)

"""Shared helpers of the parity tests: seeded inputs, oracle call, tolerance (SURVEY.md 7, 8c)."""
import numpy as np

from oracle import ref_layers as R
from tf_gnn_samples_b200 import batching, weights as W

TOL = 1e-4   # north-star tolerance: max-norm relative error of fp32 outputs vs the reference path


def tiny_graph(num_nodes=37, num_edges=(60, 0, 45, 11), seed=0, with_isolated=True, duplicates=True):
    """Small multigraph with the edge cases the reference's data paths produce (SURVEY.md 4.3):
    an empty edge type, isolated targets, duplicate edges, self loops, unsorted targets."""
    rng = np.random.default_rng(seed)
    hi = num_nodes - 3 if with_isolated else num_nodes       # last 3 nodes never appear as targets
    adj = []
    for e in num_edges:
        src = rng.integers(0, num_nodes, size=e)
        tgt = rng.integers(0, hi, size=e)
        a = np.stack([src, tgt], axis=1).astype(np.int32)
        if duplicates and e >= 4:
            a[1] = a[0]
            a[3] = a[2][::-1]
        adj.append(a.reshape(-1, 2))
    indeg = np.stack([np.bincount(a[:, 1], minlength=num_nodes) for a in adj]).astype(np.float32)
    return adj, indeg


def node_states(num_nodes, dim, seed=1):
    return np.tanh(np.random.default_rng(seed).standard_normal((num_nodes, dim))).astype(np.float32)


def assert_parity(got, want64, what="", tol=TOL):
    got = np.asarray(got, dtype=np.float64)
    want64 = np.asarray(want64, dtype=np.float64)
    assert got.shape == want64.shape, "%s: shape %s vs %s" % (what, got.shape, want64.shape)
    assert np.all(np.isfinite(got)), "%s: non-finite output" % what
    err = R.max_norm_rel_err(got, want64)
    assert err <= tol, "%s: max-norm relative error %.3e > %.1e" % (what, err, tol)
    scale = float(np.max(np.abs(want64))) if want64.size else 1.0
    assert np.allclose(got, want64, rtol=tol, atol=tol * max(scale, 1e-30)), "%s: allclose failed" % what
    return err


def to_cuda_inputs(h, adj, indeg, device):
    import torch
    return (torch.as_tensor(h).to(device),
            [torch.as_tensor(a).to(device) for a in adj],
            None if indeg is None else torch.as_tensor(indeg).to(device))


def launched_kernels(fn, expect=()):
    """Run `fn` under torch.profiler with CUDA activities and return the set of demangled names of the kernels it launched
    (CUPTI records every kernel of the process, including those launched by librgnn.so through ctypes).  A test asserts
    the variant it means to exercise is among them, so a heuristic that later routes the shape elsewhere fails loudly.

    The device trace has been seen to come back without some of the kernels a run launched (once without any).  The
    window is padded on both sides, and while a name containing one of the `expect` substrings is missing `fn` is
    profiled again, at most three times in all, so `fn` must be safe to repeat.  A kernel that is never launched is
    still missing from the result."""
    import time
    import torch
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.05)
            fn()
            torch.cuda.synchronize()
            time.sleep(0.05)
        names |= {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names and all(any(s in n for n in names) for s in expect):
            break
    return names


def assert_parity_8c(got, want64, want32, what=""):
    """SURVEY.md 8(c) acceptance, both clauses spelled out: max-norm relative error vs the float64 truth <= 1e-4 (north
    star) AND no worse than 10x the error the reference-order float32 arithmetic (`want32`) makes itself.  Deep stacks
    (timesteps x layer norm) amplify float32 rounding in the reference path too, so the second clause has a floor of 1e-5;
    both errors are printed."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == np.asarray(want64).shape, "%s: shape %s vs %s" % (what, got.shape, np.asarray(want64).shape)
    assert np.all(np.isfinite(got)), "%s: non-finite output" % what
    err = R.max_norm_rel_err(got, want64)
    err32 = R.max_norm_rel_err(np.asarray(want32, np.float64), want64)
    print("%s: engine %.2e | reference-order float32 %.2e (max-norm relative error vs float64)" % (what, err, err32))
    assert err <= TOL, "%s: max-norm relative error %.3e > %.1e (reference float32 path: %.3e)" % (what, err, TOL, err32)
    assert err <= max(10.0 * err32, 1e-5), "%s: engine error %.3e is more than 10x the reference float32 path's %.3e" % (what, err, err32)
    return err, err32

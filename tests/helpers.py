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


def rel(got, want):
    """max |got - want| / max |want| (the absolute difference when want is all zeros)."""
    want = np.asarray(want, np.float64)
    scale = np.abs(want).max()
    d = np.abs(np.asarray(got, np.float64) - want).max()
    return float(d / scale) if scale > 0 else float(d)


def to_dev(weights, device):
    """numpy weight container -> the same container of float32 leaf tensors on `device` that require a gradient."""
    import torch
    if isinstance(weights, dict):
        return {k: to_dev(v, device) for k, v in weights.items()}
    if isinstance(weights, (list, tuple)):
        return [to_dev(v, device) for v in weights]
    if weights is None:
        return None
    return torch.as_tensor(np.ascontiguousarray(weights), dtype=torch.float32).to(device).requires_grad_(True)


def compare(engine_fn, oracle_fn, h, w, proj_seed=0, tol=TOL, expect=None):
    """engine_fn(h_dev, w_dev) / oracle_fn(h64, w64) -> output; compares output and d<out, proj>/d{h, every weight} with
    torch float64 autograd over the reference op order (oracle/ref_autograd.py).  Returns ({name: error}, kernel names).

    With `expect` (kernel-name substrings, see launched_kernels) only the backward pass is profiled -- the forward runs
    outside the profiler, so every name returned was launched by a gradient -- and the kernel names are returned; without
    it the name set is empty."""
    import torch
    from oracle import ref_autograd as A
    dev = torch.device("cuda", 0)
    hd = torch.as_tensor(h).to(dev).requires_grad_(True)
    wd = to_dev(w, dev)
    out = engine_fn(hd, wd)
    proj = np.random.default_rng(proj_seed).standard_normal(tuple(out.shape)).astype(np.float32)
    loss = (out * torch.as_tensor(proj).to(dev)).sum()
    names = set()
    if expect is None:
        loss.backward()
    else:
        leaves = [hd] + list(A.flatten(wd).values())

        def backward():                       # launched_kernels may run it up to three times: start each from no gradient
            for t in leaves:
                t.grad = None
            loss.backward(retain_graph=True)
        names = launched_kernels(backward, expect)
    h64 = torch.as_tensor(h, dtype=torch.float64).requires_grad_(True)
    w64 = A.to_torch64(w)
    out64 = oracle_fn(h64, w64)
    (out64 * torch.as_tensor(proj, dtype=torch.float64)).sum().backward()
    errs = {"out": rel(out.detach().cpu().numpy(), out64.detach().numpy()), "d_h": rel(hd.grad.cpu().numpy(), h64.grad.numpy())}
    fd, f64 = A.flatten(wd), A.flatten(w64)
    assert list(fd) == list(f64)
    for k in fd:
        if f64[k].grad is None:
            assert fd[k].grad is None or float(fd[k].grad.abs().max()) == 0.0, k
            continue
        if fd[k].grad is None:                                   # e.g. the kernel of an edge type without edges: autograd never sees it
            assert float(f64[k].grad.abs().max()) == 0.0, "no gradient reached %s" % k
            continue
        errs["d_" + k] = rel(fd[k].grad.cpu().numpy(), f64[k].grad.numpy())
    print({k: "%.1e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, bad
    return errs, names


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

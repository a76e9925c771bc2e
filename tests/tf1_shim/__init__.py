"""A numpy-backed stand-in for the slice of TensorFlow 1.13 / dpu_utils that the reference calls.

TEST INFRASTRUCTURE (like oracle/): it exists so that the UNMODIFIED reference sources can be imported and executed in this
container (TF1 is not installable: Python 3.12, no network), eagerly, on numpy arrays:
  gnns/{rgcn,ggnn,rgat,gnn_film,gnn_edge_mlp,rgin,rgdcn}.py, utils/utils.py      the layer functions        (this file)
  tasks/{sparse_graph,qm9,ppi}_task.py                                            loaders, batchers, heads   (+ graph_mode.py)
  models/sparse_graph_model.py, models/*_model.py, utils/model_utils.py           scaffold, train step, epoch loop, save / restore
The reference-owned logic -- which rows are gathered, which kernel multiplies what, where the normalisation / activation /
layer norm sit, how heads, timesteps, layers and epochs are looped, which variables are created under which names, what is
logged -- then runs exactly as written; what this package restates are only the TF / Keras / dpu_utils KERNEL semantics
(SURVEY.md Appendix A), each cited where it is defined.  ``tests/golden/make_*_fixtures.py`` use it to produce the committed
fixtures; ``tests/golden/make_tf1_fixtures.py`` produces the layer fixtures with a real TensorFlow 1.13 for anyone who has one.

Usage:
    with tf1_shim.installed(dtype=np.float64, seed=0) as session:
        from gnns import sparse_rgcn_layer            # the reference's own module
        with session.tf.variable_scope("graph_model"), session.tf.variable_scope("gnn_layer_0"):
            out = sparse_rgcn_layer(h, adjacency_lists, num_incoming, state_dim=D, ...)
        session.variables                              # {"graph_model/gnn_layer_0/Edge_0_Weight/kernel:0": array, ...}
    (whole models: tests/golden/model_cases.py; batchers: tests/golden/batcher_cases.py; epoch loop: tests/test_reference_training_pin.py)

Tensors are numpy arrays; every op runs immediately.  Variables are created on first use by ``session.provider``
(default: the Keras / tf.get_variable default initialisers from a seeded generator; tests pass explicit values).
"""
import contextlib
import math
import os
import sys
import types
from typing import Callable, Dict, List, Optional

import numpy as np

# a checkout of the original microsoft/tf-gnn-samples: only the fixture generators under tests/golden execute it
REFERENCE_ROOT = os.environ.get("TF_GNN_SAMPLES_REFERENCE", "")
_F32_LOWEST = float(np.finfo(np.float32).min)


class Session:
    """State of one shim installation: dtype, variable scopes, created variables (in creation order)."""

    def __init__(self, dtype=np.float64, seed: int = 0, provider: Optional[Callable] = None):
        self.dtype = np.dtype(dtype).type
        self.rng = np.random.default_rng(seed)
        self.provider = provider
        self.scope: List[str] = []
        self.variables: Dict[str, np.ndarray] = {}
        self._uid: Dict[str, int] = {}
        self.tf = None
        self.feeds: Optional[Dict[str, np.ndarray]] = None     # graph_mode: placeholder name -> value (None: inert placeholders)
        self.non_trainable = set()
        self.run_hook: Optional[Callable] = None                # graph_mode: scripted sess.run (epoch-loop tests)
        self.gradient_hook: Optional[Callable] = None           # graph_mode: prescribed gradients (train-step tests)
        self.optimizers, self.applied, self.loss_for_gradients = [], None, None

    # -- naming (tf.variable_scope(None, default_name=...) / Keras unique layer names) --
    def scope_path(self) -> str:
        return "/".join(self.scope)

    def unique(self, base: str) -> str:
        key = self.scope_path() + "/" + base
        n = self._uid.get(key, 0)
        self._uid[key] = n + 1
        return base if n == 0 else "%s_%d" % (base, n)

    def get_variable(self, name: str, shape, init: str) -> np.ndarray:
        full = (self.scope_path() + "/" if self.scope else "") + name + ":0"
        if full in self.variables:
            return self.variables[full]
        shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        value = self.provider(full, shape, init) if self.provider is not None else None
        if value is None:
            value = self._initial_value(shape, init)
        value = np.asarray(value)
        assert value.shape == shape, "variable %s: provided shape %s != %s" % (full, value.shape, shape)
        # weights live in float32 in the reference; the float64 run uses the same float32 values widened
        value = value.astype(np.float32).astype(self.dtype)
        self.variables[full] = value
        return value

    def _initial_value(self, shape, init: str) -> np.ndarray:
        if init == "zeros":
            return np.zeros(shape, np.float32)
        if init == "ones":
            return np.ones(shape, np.float32)
        if init == "glorot_uniform":             # Keras Dense / tf.get_variable default (A.1, A.8)
            fan_in = shape[0] if len(shape) >= 1 else 1
            fan_out = shape[-1] if len(shape) >= 1 else 1
            limit = math.sqrt(6.0 / (fan_in + fan_out))
            return self.rng.uniform(-limit, limit, size=shape).astype(np.float32)
        if init == "orthogonal":                 # Keras recurrent_initializer (A.4): one orthogonal matrix of the full shape
            rows, cols = shape
            a = self.rng.standard_normal((max(rows, cols), min(rows, cols)))
            q, r = np.linalg.qr(a)
            q = q * np.sign(np.diag(r))
            return (q if rows >= cols else q.T)[:rows, :cols].astype(np.float32)
        if init.startswith("truncated_normal:"):
            sd = float(init.split(":")[1])
            return (np.clip(self.rng.standard_normal(shape), -2.0, 2.0) * sd).astype(np.float32)
        raise ValueError("unknown initialiser %r" % init)


# ---------------------------------------------------------------------------------------------------------------
# op restatements (TF 1.13 kernel semantics)
# ---------------------------------------------------------------------------------------------------------------
def _segment_sum(data, segment_ids, num_segments):
    """tf.unsorted_segment_sum (A.2): zeros for empty segments; CPU kernel accumulates in message order."""
    data = np.asarray(data)
    out = np.zeros((int(num_segments),) + data.shape[1:], dtype=data.dtype)
    np.add.at(out, np.asarray(segment_ids), data)
    return out


def _segment_count(data, segment_ids, num_segments):
    n = np.bincount(np.asarray(segment_ids), minlength=int(num_segments)).astype(data.dtype)
    return np.maximum(n, data.dtype.type(1)).reshape((-1,) + (1,) * (data.ndim - 1))


def _segment_mean(data, segment_ids, num_segments):
    """tf.unsorted_segment_mean = sum / max(count, 1) (math_ops.py: _unsorted_segment_N)."""
    data = np.asarray(data)
    return _segment_sum(data, segment_ids, num_segments) / _segment_count(data, segment_ids, num_segments)


def _segment_sqrt_n(data, segment_ids, num_segments):
    """tf.unsorted_segment_sqrt_n = sum / sqrt(max(count, 1))."""
    data = np.asarray(data)
    return _segment_sum(data, segment_ids, num_segments) / np.sqrt(_segment_count(data, segment_ids, num_segments))


def _segment_max(data, segment_ids, num_segments):
    """tf.unsorted_segment_max: empty segment = numeric_limits<float>::lowest() (the reference computes in float32)."""
    data = np.asarray(data)
    out = np.full((int(num_segments),) + data.shape[1:], _F32_LOWEST, dtype=data.dtype)
    np.maximum.at(out, np.asarray(segment_ids), data)
    return out


def _erf(x):
    from scipy.special import erf
    return erf(x).astype(np.asarray(x).dtype)


def _elu(x):
    x = np.asarray(x)
    return np.where(x > 0, x, np.expm1(np.minimum(x, x.dtype.type(0))))


def _selu(x):
    x = np.asarray(x)
    scale, alpha = x.dtype.type(1.0507009873554805), x.dtype.type(1.6732632423543772)
    return scale * np.where(x > 0, x, alpha * np.expm1(np.minimum(x, x.dtype.type(0))))


def _leaky_relu(x, alpha=0.2):
    x = np.asarray(x)
    return np.where(x > 0, x, x * x.dtype.type(alpha))       # tf.nn.leaky_relu default alpha = 0.2


def _hard_sigmoid(x):
    t = x.dtype.type
    return np.clip(t(0.2) * x + t(0.5), t(0), t(1))          # keras.backend.hard_sigmoid


def build_modules(session: Session):
    """Return {module name: module} for 'tensorflow', 'dpu_utils', 'dpu_utils.tfutils'."""
    tf = types.ModuleType("tensorflow")
    tf.__shim__ = True
    tf.Tensor = np.ndarray
    tf.int32, tf.int64, tf.float32, tf.float64 = np.int32, np.int64, np.float32, np.float64

    def shape(x, out_type=None, name=None):
        return np.asarray(np.asarray(x).shape, dtype=out_type or np.int32)

    tf.shape = shape
    tf.concat = lambda values, axis, name=None: np.concatenate([np.asarray(v) for v in values], axis=axis) \
        if not isinstance(values, np.ndarray) else np.asarray(values)   # rgat.py:126 passes ONE tensor: concat is the identity
    tf.expand_dims = lambda x, axis=None, name=None: np.expand_dims(np.asarray(x), axis)
    tf.reshape = lambda x, shape, name=None: np.reshape(np.asarray(x), tuple(int(s) for s in shape))
    tf.einsum = lambda eq, *ops: np.einsum(eq, *ops)
    tf.exp, tf.log, tf.tanh, tf.sqrt = np.exp, np.log, np.tanh, lambda x: np.sqrt(session.dtype(x) if np.isscalar(x) else x)
    tf.erf = _erf
    tf.round, tf.cast = np.round, lambda x, dtype: np.asarray(x).astype(dtype)
    tf.count_nonzero = np.count_nonzero
    tf.unsorted_segment_sum = lambda data, segment_ids, num_segments, name=None: _segment_sum(data, segment_ids, num_segments)
    tf.unsorted_segment_max = lambda data, segment_ids, num_segments, name=None: _segment_max(data, segment_ids, num_segments)
    tf.unsorted_segment_mean = lambda data, segment_ids, num_segments, name=None: _segment_mean(data, segment_ids, num_segments)
    tf.unsorted_segment_sqrt_n = lambda data, segment_ids, num_segments, name=None: _segment_sqrt_n(data, segment_ids, num_segments)
    tf.gather = lambda params, indices, name=None: np.asarray(params)[np.asarray(indices)]

    @contextlib.contextmanager
    def variable_scope(name_or_scope, default_name=None, reuse=None):
        name = name_or_scope if name_or_scope is not None else session.unique(default_name)
        session.scope.append(name)
        try:
            yield name
        finally:
            session.scope.pop()

    tf.variable_scope = variable_scope

    def get_variable(name, shape=None, dtype=None, initializer=None, trainable=True):
        # default initializer of tf.get_variable for float variables: glorot_uniform_initializer (A.8)
        return session.get_variable(name, shape, "glorot_uniform")

    tf.get_variable = get_variable

    nn = types.ModuleType("tensorflow.nn")
    nn.embedding_lookup = lambda params, ids, name=None: np.asarray(params)[np.asarray(ids)]
    nn.relu = lambda x, name=None: np.maximum(x, np.asarray(x).dtype.type(0))
    nn.leaky_relu = _leaky_relu
    nn.elu, nn.selu = _elu, _selu
    nn.sigmoid = lambda x: 1.0 / (1.0 + np.exp(-x))

    def dropout(x, keep_prob=None, rate=None, **kw):
        if rate is None:
            rate = 0.0 if keep_prob is None else 1.0 - keep_prob
        assert float(rate) == 0.0, "the shim only runs the evaluation path (dropout rate 0 = identity, A.9)"
        return x

    nn.dropout = dropout
    tf.nn = nn

    class _Dense:
        """tf.keras.layers.Dense / tf.layers.Dense: y = activation(x @ kernel [+ bias]), kernel [in, units] Glorot-uniform (A.1)."""
        _default_name = "dense"

        def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None, name=None, **kw):
            self.units, self.activation, self.use_bias, self.name = int(units), activation, use_bias, name
            self.kernel_init = kernel_initializer or "glorot_uniform"
            self.kernel = self.bias = None

        def __call__(self, inputs):
            inputs = np.asarray(inputs)
            if self.kernel is None:
                if self.name is None:
                    self.name = session.unique(self._default_name)
                session.scope.append(self.name)
                try:
                    self.kernel = session.get_variable("kernel", (inputs.shape[-1], self.units), self.kernel_init)
                    if self.use_bias:
                        self.bias = session.get_variable("bias", (self.units,), "zeros")
                finally:
                    session.scope.pop()
            y = inputs @ self.kernel.astype(inputs.dtype)
            if self.bias is not None:
                y = y + self.bias.astype(inputs.dtype)
            return y if self.activation is None else self.activation(y)

    class _SimpleRNNCell:
        """tf.keras.layers.SimpleRNNCell: h' = activation(x.W + b + h.U); returns (h', [h']) (A.4)."""

        def __init__(self, units, activation=None, **kw):
            self.units, self.activation, self.built = int(units), activation, False

        def _build(self, in_dim):
            name = session.unique("simple_rnn_cell")
            session.scope.append(name)
            try:
                self.kernel = session.get_variable("kernel", (in_dim, self.units), "glorot_uniform")
                self.recurrent_kernel = session.get_variable("recurrent_kernel", (self.units, self.units), "orthogonal")
                self.bias = session.get_variable("bias", (self.units,), "zeros")
            finally:
                session.scope.pop()
            self.built = True

        def __call__(self, inputs, states):
            inputs, h = np.asarray(inputs), np.asarray(states[0])
            if not self.built:
                self._build(inputs.shape[-1])
            out = (inputs @ self.kernel + self.bias) + h @ self.recurrent_kernel
            out = out if self.activation is None else self.activation(out)
            return out, [out]

    class _GRUCell:
        """tf.keras.layers.GRUCell with the TF 1.13 defaults (A.4): recurrent_activation = hard_sigmoid, use_bias,
        reset_after = False, implementation 1; kernels [in, 3u] / [u, 3u] / [3u] in gate order z | r | h."""

        def __init__(self, units, activation=None, **kw):
            self.units, self.activation, self.built = int(units), activation, False

        def _build(self, in_dim):
            name = session.unique("gru_cell")
            session.scope.append(name)
            try:
                u = self.units
                self.kernel = session.get_variable("kernel", (in_dim, 3 * u), "glorot_uniform")
                self.recurrent_kernel = session.get_variable("recurrent_kernel", (u, 3 * u), "orthogonal")
                self.bias = session.get_variable("bias", (3 * u,), "zeros")
            finally:
                session.scope.pop()
            self.built = True

        def __call__(self, inputs, states):
            inputs, h = np.asarray(inputs), np.asarray(states[0])
            if not self.built:
                self._build(inputs.shape[-1])
            u, k, rk, b = self.units, self.kernel, self.recurrent_kernel, self.bias
            x_z = inputs @ k[:, :u] + b[:u]
            x_r = inputs @ k[:, u:2 * u] + b[u:2 * u]
            x_h = inputs @ k[:, 2 * u:] + b[2 * u:]
            z = _hard_sigmoid(x_z + h @ rk[:, :u])
            r = _hard_sigmoid(x_r + h @ rk[:, u:2 * u])
            hh = x_h + (r * h) @ rk[:, 2 * u:]
            hh = hh if self.activation is None else self.activation(hh)
            out = z * h + (inputs.dtype.type(1) - z) * hh
            return out, [out]

    class _LSTMCell:
        def __init__(self, units, activation=None, **kw):
            self.units = units

        def __call__(self, inputs, states):
            # Keras unpacks h_tm1, c_tm1 = states[0], states[1]; the reference passes ONE state (ggnn.py:92)
            raise ValueError("LSTMCell expects states [h, c]; got %d state(s)" % len(states))

    keras = types.ModuleType("tensorflow.keras")
    keras.layers = types.ModuleType("tensorflow.keras.layers")

    class _KerasDense(_Dense):
        """tf.keras.layers.Dense: an unnamed Keras layer takes its name at CONSTRUCTION from a per-graph counter that ignores
        scopes (backend.unique_object_name: dense, dense_1, ...), whereas an unnamed tf.layers.Dense opens
        variable_scope(None, default_name='dense') at its first call and is numbered within the enclosing scope."""

        def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None, name=None, **kw):
            if name is None:
                n = session._uid.get("<keras>/dense", 0)
                session._uid["<keras>/dense"] = n + 1
                name = "dense" if n == 0 else "dense_%d" % n
            super().__init__(units, activation, use_bias, kernel_initializer, name, **kw)

    keras.layers.Dense = _KerasDense
    keras.layers.SimpleRNNCell, keras.layers.GRUCell, keras.layers.LSTMCell = _SimpleRNNCell, _GRUCell, _LSTMCell
    tf.keras = keras
    layers = types.ModuleType("tensorflow.layers")
    layers.Dense = _Dense
    tf.layers = layers

    initializers = types.ModuleType("tensorflow.initializers")
    initializers.truncated_normal = lambda mean=0.0, stddev=1.0, **kw: "truncated_normal:%r" % float(stddev)
    tf.initializers = initializers

    def layer_norm(inputs, center=True, scale=True, begin_norm_axis=1, begin_params_axis=-1, scope=None, **kw):
        """tf.contrib.layers.layer_norm defaults (A.5): moments over axes [1, rank), biased variance, variance_epsilon
        1e-12, evaluated by tf.nn.batch_normalization as x*inv + (beta - mean*inv), inv = rsqrt(var + eps) * gamma;
        variables 'beta' (zeros) then 'gamma' (ones) of shape [D] under variable_scope(scope, 'LayerNorm')."""
        inputs = np.asarray(inputs)
        with variable_scope(scope, default_name="LayerNorm"):
            beta = session.get_variable("beta", (inputs.shape[-1],), "zeros")
            gamma = session.get_variable("gamma", (inputs.shape[-1],), "ones")
        t = inputs.dtype.type
        mean = inputs.mean(axis=-1, keepdims=True)
        var = ((inputs - mean) ** 2).mean(axis=-1, keepdims=True)
        inv = (t(1) / np.sqrt(var + t(1e-12))) * gamma.astype(inputs.dtype)
        return inputs * inv + (beta.astype(inputs.dtype) - mean * inv)

    contrib = types.ModuleType("tensorflow.contrib")
    contrib.layers = types.ModuleType("tensorflow.contrib.layers")
    contrib.layers.layer_norm = layer_norm
    tf.contrib = contrib

    dpu = types.ModuleType("dpu_utils")
    tfutils = types.ModuleType("dpu_utils.tfutils")

    def unsorted_segment_log_softmax(logits, segment_ids, num_segments):
        """dpu_utils.tfutils.unsorted_segment_log_softmax (dpu-utils >= 0.1.30, A.7): segment max, recentre, exp,
        segment sum, log, subtract -- composed from the same tf ops."""
        max_per_segment = tf.unsorted_segment_max(data=logits, segment_ids=segment_ids, num_segments=num_segments)
        scattered_maxes = tf.gather(params=max_per_segment, indices=segment_ids)
        recentered_scores = logits - scattered_maxes
        exped_recentered_scores = tf.exp(recentered_scores)
        per_segment_sums = tf.unsorted_segment_sum(exped_recentered_scores, segment_ids, num_segments)
        with np.errstate(divide="ignore"):
            per_segment_normalization_consts = tf.log(per_segment_sums)
        return recentered_scores - tf.gather(params=per_segment_normalization_consts, indices=segment_ids)

    tfutils.unsorted_segment_log_softmax = unsorted_segment_log_softmax
    dpu.tfutils = tfutils

    class RichPath:
        """dpu_utils.utils.RichPath, local files only: what the reference's loaders call (tasks/qm9_task.py:77-87,
        tasks/ppi_task.py:85-88) -- join, .path, read_by_file_suffix for .jsonl.gz (generator of records), .json, .npy."""

        def __init__(self, path):
            self.path = str(path)

        @classmethod
        def create(cls, path, azure_info_path=None):
            return cls(path)

        def join(self, filename):
            return RichPath(os.path.join(self.path, filename))

        def __str__(self):
            return self.path

        __repr__ = __str__

        def read_by_file_suffix(self):
            import gzip
            import json
            if self.path.endswith(".jsonl.gz"):
                def records():
                    with gzip.open(self.path, "rt") as f:
                        for line in f:
                            yield json.loads(line)
                return records()
            if self.path.endswith(".json"):
                with open(self.path) as f:
                    return json.load(f)
            if self.path.endswith(".npy"):
                return np.load(self.path)
            raise ValueError("unsupported suffix: %s" % self.path)

    from . import graph_mode
    dpu_utils_utils = types.ModuleType("dpu_utils.utils")
    dpu_utils_utils.RichPath = RichPath
    dpu_utils_utils.ThreadedIterator = graph_mode.ThreadedIterator
    dpu.utils = dpu_utils_utils
    extra = graph_mode.extend(tf, session)       # placeholders, Graph / Session, optimizers, summaries, head ops
    session.tf = tf
    return {**extra, "tensorflow": tf, "dpu_utils.utils": dpu_utils_utils, "tensorflow.nn": nn, "tensorflow.keras": keras, "tensorflow.keras.layers": keras.layers,
            "tensorflow.layers": layers, "tensorflow.contrib": contrib, "tensorflow.contrib.layers": contrib.layers,
            "tensorflow.initializers": initializers, "dpu_utils": dpu, "dpu_utils.tfutils": tfutils}


_REFERENCE_MODULES = ("gnns", "utils", "tasks", "models")


def import_reference_task(module: str, reference_root: str = REFERENCE_ROOT):
    """Import the reference's ``tasks/<module>.py`` inside an ``installed()`` block WITHOUT running tasks/__init__.py (it
    pulls in the VarMisuse task and with it dpu_utils.codeutils, which the shim does not restate): a bare package object
    with the right __path__ stands in for it, the submodule itself is the unmodified reference file."""
    import importlib
    if "tasks" not in sys.modules:
        pkg = types.ModuleType("tasks")
        pkg.__path__ = [os.path.join(reference_root, "tasks")]
        sys.modules["tasks"] = pkg
        base = importlib.import_module("tasks.sparse_graph_task")      # what models/sparse_graph_model.py:12 imports from 'tasks'
        pkg.Sparse_Graph_Task, pkg.DataFold = base.Sparse_Graph_Task, base.DataFold
    mod = importlib.import_module("tasks." + module)
    assert os.path.realpath(mod.__file__).startswith(os.path.realpath(reference_root)), mod.__file__
    return mod


def import_reference_model_utils(reference_root: str = REFERENCE_ROOT):
    """The reference's utils/model_utils.py (name_to_model_class, name_to_task_class, restore) inside an ``installed()`` block.
    It imports four task classes from ``tasks``; the two whose modules the shim cannot load (Citation_Network_Task: scipy
    loaders are fine but unused here; VarMisuse_Task: dpu_utils.codeutils) are present as None."""
    import importlib
    qm9, ppi = import_reference_task("qm9_task", reference_root), import_reference_task("ppi_task", reference_root)
    pkg = sys.modules["tasks"]
    pkg.QM9_Task, pkg.PPI_Task = qm9.QM9_Task, ppi.PPI_Task
    pkg.Citation_Network_Task = pkg.VarMisuse_Task = None
    return importlib.import_module("utils.model_utils")


@contextlib.contextmanager
def installed(dtype=np.float64, seed: int = 0, provider: Optional[Callable] = None, reference_root: str = REFERENCE_ROOT):
    """Install the shim as ``tensorflow`` / ``dpu_utils`` and put the reference on sys.path for the duration of the
    block; the reference's ``gnns`` / ``utils`` packages are imported fresh (bound to THIS session) and removed again
    afterwards, so nothing leaks into other tests."""
    session = Session(dtype, seed, provider)
    mods = build_modules(session)
    saved = {k: sys.modules.get(k) for k in list(mods) + [m for m in list(sys.modules)
                                                             if m.split(".")[0] in _REFERENCE_MODULES]}
    for k in list(sys.modules):
        if k.split(".")[0] in _REFERENCE_MODULES:
            del sys.modules[k]
    sys.modules.update(mods)
    if reference_root:
        sys.path.insert(0, reference_root)
    import warnings
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SyntaxWarning)   # the reference's docstrings hold '\e' escapes (Python 3.12 warns)
            yield session
    finally:
        if reference_root:
            sys.path.remove(reference_root)
        for k in list(sys.modules):
            if k.split(".")[0] in _REFERENCE_MODULES or k in mods:
                del sys.modules[k]
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v

"""Host mirror of the reference's utils/utils.py factories.

The reference returns TF callables; here the same names return the enum codes the C ABI takes
(include/rgnn.h), with the reference's error behaviour: ValueError for unknown activation /
aggregation names (utils/utils.py:33,58), Exception for an unknown cell (utils/utils.py:20).
"""
from typing import Optional

BIG_NUMBER = 1e7      # utils/utils.py:6
SMALL_NUMBER = 1e-7   # utils/utils.py:7  (baked into the kernels as 1e-7f)

ACT_LINEAR, ACT_TANH, ACT_RELU, ACT_LEAKY_RELU, ACT_ELU, ACT_SELU, ACT_GELU = range(7)
AGG_SUM, AGG_MAX, AGG_MEAN, AGG_SQRT_N = range(4)
CELL_RNN, CELL_GRU = range(2)
LAYER_RGCN, LAYER_GGNN, LAYER_RGAT, LAYER_FILM, LAYER_EDGE_MLP, LAYER_RGIN, LAYER_RGCN_BACKWARD, LAYER_RGDCN = range(8)
LAYER_FILM_BACKWARD = 8   # rgnn_workspace_bytes of rgnn_film_backward
LAYER_RGAT_BACKWARD = 9   # rgnn_workspace_bytes of rgnn_rgat_backward
LAYER_GGNN_BACKWARD = 10  # rgnn_workspace_bytes of rgnn_ggnn_backward
LAYER_RGIN_BACKWARD = 11  # rgnn_workspace_bytes of rgnn_rgin_backward
LAYER_RGDCN_BACKWARD = 12  # rgnn_workspace_bytes of rgnn_rgdcn_backward (pass channel_dim as mlp_layers)

_ACTIVATIONS = {"linear": ACT_LINEAR, "tanh": ACT_TANH, "relu": ACT_RELU, "leaky_relu": ACT_LEAKY_RELU,
                "elu": ACT_ELU, "selu": ACT_SELU, "gelu": ACT_GELU}


def get_activation(activation_fun: Optional[str]) -> int:
    """utils/utils.py:36-58.  None / 'linear' -> identity (the reference returns None there; where it
    would then call None(...) and crash, this engine applies the identity -- a documented superset)."""
    if activation_fun is None:
        return ACT_LINEAR
    name = activation_fun.lower()
    if name not in _ACTIVATIONS:
        raise ValueError("Unknown activation function '%s'!" % activation_fun)
    return _ACTIVATIONS[name]


def get_aggregation_function(aggregation_fun: Optional[str]) -> int:
    """utils/utils.py:23-33 (names are case-sensitive there too)."""
    if aggregation_fun in ['sum', 'unsorted_segment_sum']:
        return AGG_SUM
    if aggregation_fun in ['max', 'unsorted_segment_max']:
        return AGG_MAX
    if aggregation_fun in ['mean', 'unsorted_segment_mean']:
        return AGG_MEAN
    if aggregation_fun in ['sqrt_n', 'unsorted_segment_sqrt_n']:
        return AGG_SQRT_N
    raise ValueError("Unknown aggregation function '%s'!" % aggregation_fun)


def get_gated_unit(units: int, gated_unit: str, activation_function: Optional[str]):
    """utils/utils.py:10-20 -> (cell code, activation code).  LSTM cannot work in the reference
    (ggnn.py:92 passes a single state to an LSTMCell) and is rejected here explicitly."""
    act = get_activation(activation_function)
    name = gated_unit.lower()
    if name == 'rnn':
        return CELL_RNN, act
    if name == 'gru':
        return CELL_GRU, act
    if name == 'lstm':
        raise NotImplementedError("LSTMCell needs [h, c] states; the reference passes one state (gnns/ggnn.py:92) "
                                  "and fails at graph construction, so there is no behaviour to reproduce")
    raise Exception("Unknown RNN cell type '%s'." % gated_unit)

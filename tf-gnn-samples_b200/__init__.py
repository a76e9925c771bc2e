"""b200-rgnn: H100-native relational GNN message passing behind the tf-gnn-samples layer API.

Host code is Python over a C-ABI CUDA library (lib/librgnn.so, include/rgnn.h); torch tensors are
the device-memory container.  There is NO CPU fallback: importing the layer functions works
anywhere, calling them requires the CUDA library and a GPU and fails loudly otherwise.
"""
from .utils import (SMALL_NUMBER, BIG_NUMBER, get_activation, get_aggregation_function,  # noqa: F401
                    get_gated_unit)
from .engine import GraphPlan, RgnnError, launch_count, set_weight_cache, weight_cache_clear  # noqa: F401
from .gnns import (sparse_rgcn_layer, sparse_ggnn_layer, sparse_rgat_layer, sparse_rgin_layer,  # noqa: F401
                   sparse_gnn_edge_mlp_layer, sparse_gnn_film_layer, sparse_rgdcn_layer, rgcn_layer_stack)

from .sharded import ShardedGraph, PeerBuffer, degree_balanced_cuts  # noqa: F401

__version__ = "0.2.0"

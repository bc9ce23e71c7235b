# coding=utf-8
"""OOP API (the subset of tf_geometric.layers on the message-passing hot path; SURVEY.md section 8b)."""
from .conv.gcn import GCN
from .conv.gat import GAT
from .conv.graph_sage import MeanGraphSage, SumGraphSage, GCNGraphSage, MeanPoolGraphSage, MaxPoolGraphSage, \
    LSTMGraphSage
from .conv.appnp import APPNP
from .conv.propagation import SGC, SSGC, TAGCN, GIN, LEConv, ChebyNet
from .pool.pool import MeanPool, SumPool, MaxPool, MinPool, Set2Set, SAGPool, SortPool
from .pool.cluster_pool import DiffPool, MinCutPool
from .pool.asap import ASAP
from .sampling import DropEdge
from .kernel import MapReduceGNN

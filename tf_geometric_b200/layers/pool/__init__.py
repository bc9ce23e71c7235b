# coding=utf-8
from .pool import MeanPool, SumPool, MaxPool, MinPool, Set2Set, SAGPool, SortPool
from .cluster_pool import DiffPool, MinCutPool
from .asap import ASAP

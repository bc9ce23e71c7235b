# coding=utf-8
from . import common_pool, set2set, topk_pool, score_pool, cluster_pool, diff_pool, min_cut_pool, asap

# coding=utf-8
from . import predict_edge

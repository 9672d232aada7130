"""Architectures of the reference expressed in the layer-list IR of graph.py."""
from . import cifar_resnet, plainnet, resnet50, resnet_v1, wide_residual_network  # noqa: F401

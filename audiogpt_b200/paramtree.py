"""Build an nn.Module parameter tree from a {dotted.key: shape} table.

The drop-in classes keep the reference's ``state_dict`` key layouts (SURVEY.md
8b) without re-declaring the reference's layer objects: parameters are plain
``nn.Parameter`` leaves hung on anonymous container modules, created from the
tables in :mod:`audiogpt_b200.specs`.  The modules are *storage only* -- all
arithmetic happens in libagpt_b200.so.
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch
from torch import nn


class ParamNode(nn.Module):
    """Anonymous container; children are ParamNodes or nn.Parameters."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("ParamNode is storage only; call the owning model")


def _descend(root: nn.Module, parts):
    node = root
    for p in parts:
        nxt = node._modules.get(p)
        if nxt is None:
            nxt = ParamNode()
            node.add_module(p, nxt)
        node = nxt
    return node


def add_param(root: nn.Module, key: str, value: torch.Tensor):
    """Hang ``value`` at ``key``; an nn.Parameter is registered as is (a parameter shared under two keys)."""
    parts = key.split(".")
    node = _descend(root, parts[:-1])
    node.register_parameter(parts[-1], value if isinstance(value, nn.Parameter) else nn.Parameter(value, requires_grad=False))


def del_param(root: nn.Module, key: str):
    parts = key.split(".")
    node = _descend(root, parts[:-1])
    del node._parameters[parts[-1]]


def add_buffer(root: nn.Module, key: str, value: torch.Tensor):
    parts = key.split(".")
    _descend(root, parts[:-1]).register_buffer(parts[-1], value)


def _leaf(root: nn.Module, key: str):
    parts = key.split(".")
    node = root
    for p in parts[:-1]:
        node = node._modules[p]
    return node, parts[-1]


def get_param(root: nn.Module, key: str) -> torch.Tensor:
    node, name = _leaf(root, key)
    return node._parameters[name]


def get_tensor(root: nn.Module, key: str) -> torch.Tensor:
    """The parameter or, failing that, the buffer at ``key``."""
    node, name = _leaf(root, key)
    t = node._parameters.get(name)
    return t if t is not None else node._buffers[name]


def build(root: nn.Module, shapes: Dict[str, Sequence[int]], init=None):
    for key, shape in shapes.items():
        t = torch.zeros(tuple(shape), dtype=torch.float32) if init is None else init(key, tuple(shape))
        add_param(root, key, t)

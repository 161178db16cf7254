"""TEST INFRASTRUCTURE ONLY -- CPU emulation of the bf16x3 training step (dim_train_set_precision(DIM_PREC_BF16X3)).

oracle/train_oracle.graph(..., emulate_bf16=True) rounds what the bf16 step stores -- tensor-core operand weights, every
stored activation and every activation gradient -- with `t.bfloat16().float()`.  The bf16x3 step stores the same values as
bf16 hi / lo pairs, i.e. rounded to hi + lo with hi = bf16(t), lo = bf16(t - hi) (about 16 significant bits); its three
tensor-core passes drop only the lo*lo product (2^-16 relative), which the emulation ignores.  graph() below runs the oracle
with exactly that rounding in place of the bf16 one and fp32 accumulation everywhere, so its deviation from the fp32 run is
the intrinsic cost of the pair storage; tests/test_train_bf16x3_emulation.py records it, tests/test_gpu_train_bf16x3.py
takes its tolerances from it."""
from __future__ import annotations

import contextlib

import torch

from oracle import train_oracle as T


def round_pair(t):
    """t rounded to the value of its bf16 hi / lo pair (hi + lo is exact in fp32)"""
    hi = t.to(torch.bfloat16).float()
    return hi + (t - hi).to(torch.bfloat16).float()


def _pair_rounding_of(self):
    # stands in for Tensor.bfloat16 while graph() runs: x.bfloat16().float() then yields round_pair(x) (a float32 tensor, so
    # .float() is the identity) with the straight-through gradient of the bf16 cast it replaces
    d = self.detach()
    return self + (round_pair(d) - d)


@contextlib.contextmanager
def _pair_storage():
    orig = torch.Tensor.bfloat16
    torch.Tensor.bfloat16 = _pair_rounding_of
    try:
        yield
    finally:
        torch.Tensor.bfloat16 = orig


def graph(weights, zin, labels, requires_grad=True, num_threads=None):
    """train_oracle.graph with the bf16x3 step's storage emulated (returns (outputs, grads) like it)"""
    with _pair_storage():
        return T.graph(weights, zin, labels, requires_grad, num_threads, emulate_bf16=True)

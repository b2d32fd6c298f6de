"""The fp64 fixed-routing reference of ``ops.moe`` that ``test_gpu_moe_reference.py`` holds the kernels to, checked
without a GPU: on tokens whose routing has no near-tie it equals ``ops.reference.moe`` (fp32) in y, psum and every
gradient; the explicit per-expert pass behind the running-error bound computes the same values as autograd; and each
wiring mistake of the self-test moves some output by more than the bound allows."""
import math

import torch

from distributed_training_guide_b200.ops import reference as ref
from test_gpu_moe_reference import MUTATIONS, PATH_SLACK, U, _path_bound, moe_fixed_grads

NAMES = ("y", "psum", "dx", "d_gate", "d_gate_up", "d_down")


def _inputs(T=160, E=8, k=2, H=64, I=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    f64 = torch.float64
    x = torch.randn(T, H, generator=g, dtype=f64)
    gate_w = torch.randn(E, H, generator=g, dtype=f64) / math.sqrt(H)
    gate_up = torch.randn(E, 2 * I, H, generator=g, dtype=f64) / math.sqrt(H)
    down = torch.randn(E, H, I, generator=g, dtype=f64) / math.sqrt(I)
    # keep the tokens whose k-th and (k+1)-th probabilities are well apart, so fp32 and fp64 choose the same experts
    top = torch.softmax(x @ gate_w.t(), -1).topk(k + 1, dim=-1).values
    x = x[(top[:, k - 1] - top[:, k]) > 1e-3]
    dy = torch.randn(x.shape[0], H, generator=g, dtype=f64)
    dpsum = torch.randn(E, generator=g, dtype=f64) * math.sqrt(H)
    idx = torch.softmax(x @ gate_w.t(), -1).topk(k, dim=-1).indices
    return x, gate_w, gate_up, down, k, dy, dpsum, idx


def test_fixed_routing_reference_equals_ops_reference():
    x, gate_w, gate_up, down, k, dy, dpsum, idx = _inputs()
    assert x.shape[0] > 100
    got = dict(zip(NAMES, moe_fixed_grads(x, gate_w, gate_up, down, idx, dy, dpsum)))
    leaves = [t.float().requires_grad_() for t in (x, gate_w, gate_up, down)]
    y, p = ref.moe(*leaves, k)
    grads = torch.autograd.grad((y, p.sum(0)), leaves, (dy.float(), dpsum.float()))
    want = dict(zip(NAMES, (y.detach(), p.sum(0).detach()) + grads))
    for n in NAMES:
        scale = want[n].abs().max().item()
        torch.testing.assert_close(got[n], want[n].double(), rtol=1e-4, atol=1e-5 * scale, msg=n)


def test_bound_pass_values_equal_autograd():
    x, gate_w, gate_up, down, k, dy, dpsum, idx = _inputs(seed=1)
    auto = dict(zip(NAMES, moe_fixed_grads(x, gate_w, gate_up, down, idx, dy, dpsum)))
    p = torch.softmax(x @ gate_w.t(), -1)
    explicit = _path_bound(x, gate_w, gate_up, down, idx, p, dy, dpsum, torch.float64)
    for n, (value, bound) in explicit.items():
        torch.testing.assert_close(value, auto[n], rtol=1e-10, atol=1e-12, msg=n)
        assert bool((bound >= value.abs()).all()), n


def test_bound_rejects_each_wiring_mistake():
    x, gate_w, gate_up, down, k, dy, dpsum, idx = _inputs(seed=2)
    base = dict(zip(NAMES, moe_fixed_grads(x, gate_w, gate_up, down, idx, dy, dpsum)))
    p = torch.softmax(x @ gate_w.t(), -1)
    bounds = _path_bound(x, gate_w, gate_up, down, idx, p, dy, dpsum, torch.float64)
    for m in MUTATIONS:
        bad = dict(zip(NAMES, moe_fixed_grads(x, gate_w, gate_up, down, idx, dy, dpsum, mutate=m)))
        # a kernel within the bound of the correct graph is more than a bound away from the mistaken one somewhere
        caught = [n for n, (_, b) in bounds.items() if ((bad[n] - base[n]).abs() > 2 * U * PATH_SLACK * b).any()]
        assert caught, m

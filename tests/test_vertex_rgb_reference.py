"""The fp64 reference of the per-vertex export colour (tests/helpers/vertex_rgb_ref.py) without a GPU: its SH4 and colour network
against the oracle (oracle/sh.py, oracle/mlp.py), its SH4 Lipschitz constant, and its per-entry bound -- an fp32 stand-in of the kernel's
arithmetic passes, and each planted fault fails."""
import pytest
import torch

from helpers import radiance_ref as rr
from helpers import vertex_rgb_ref as vr
from oracle import mlp as omlp
from oracle import sh as osh


def _dirs(n, seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    return d / d.norm(dim=-1, keepdim=True)


def _inputs(n, seed, n_feat=13):
    g = torch.Generator().manual_seed(seed)
    feat = (torch.rand(n, n_feat, generator=g) * 2 - 1) * 0.8
    grad = torch.randn(n, 3, generator=g) * torch.exp2(torch.randint(-6, 8, (n, 1), generator=g).float())
    return feat, grad


def test_sh4_is_the_oracle_basis():
    d = _dirs(1000, 0)
    assert torch.allclose(vr.sh4(d), osh.sh4((d + 1) / 2), rtol=0, atol=1e-14)


def test_sh4_lipschitz_constant():
    d = _dirs(20000, 1) * 1.01
    h = 1e-6
    jac = torch.stack([(vr.sh4(d + h * torch.eye(3, dtype=torch.float64)[j]) - vr.sh4(d - h * torch.eye(3, dtype=torch.float64)[j])) / (2 * h)
                       for j in range(3)], -1)
    assert float(jac.abs().sum(-1).max()) < vr.SH_LIP


def test_network_is_the_oracle_mlp():
    params16, _ = rr.make_params(3)
    feat, grad = _inputs(500, 2)
    X, _ = vr.rows(feat.double(), grad.double())
    ours, _ = vr.forward(feat.double(), params16, None, 0, grad=grad.double())
    ref = omlp.ffmlp_fwd(X, params16.double(), 32, 3, 64, 2, emulate_fp16=False, compute_dtype=torch.float64)
    assert torch.allclose(ours, ref, rtol=0, atol=1e-12)
    # the fixed NeRF direction: [feature 16 | SH4(0, 0, -1)]
    f16, _ = _inputs(100, 4, n_feat=16)
    X, _ = vr.rows(f16.double(), fixed_dir=(0.0, 0.0, -1.0))
    sh = osh.sh4(torch.tensor([[0.5, 0.5, 0.0]], dtype=torch.float64)).expand(100, 16)
    assert torch.equal(X, torch.cat([f16.double(), sh], -1))


CASES = [(False, 1), (False, 2), (False, 0), (True, 2), (True, 0)]


@pytest.mark.parametrize('vanilla,act_mode', CASES)
def test_the_standin_passes_the_bound(vanilla, act_mode):
    params16, bias = rr.make_params(5, vanilla=vanilla)
    feat, grad = _inputs(4000, 6)
    ref, B = vr.forward(feat.double(), params16, bias, act_mode, grad=grad.double())
    worst = vr.check(vr.standin(feat, params16, bias, act_mode, grad=grad), ref, B, f'vanilla {vanilla} mode {act_mode}')
    assert worst <= 1.0
    f16, _ = _inputs(1000, 7, n_feat=16)
    ref, B = vr.forward(f16.double(), params16, bias, act_mode, fixed_dir=(0.0, 0.0, -1.0))
    vr.check(vr.standin(f16, params16, bias, act_mode, fixed_dir=(0.0, 0.0, -1.0)), ref, B, 'fixed direction')


@pytest.mark.parametrize('fault', ['view_along_normal', 'unnormalised', 'sh_of_unit_cube', 'no_bias', 'no_activation'])
def test_planted_faults_fail_the_bound(fault):
    vanilla = fault == 'no_bias'
    params16, bias = rr.make_params(5, vanilla=vanilla)
    if vanilla:
        bias = bias * 4
    feat, grad = _inputs(4000, 6)
    ref, B = vr.forward(feat.double(), params16, bias, 2, grad=grad.double())
    with pytest.raises(AssertionError, match='outside the bound'):
        vr.check(vr.standin(feat, params16, bias, 2, grad=grad, fault=fault), ref, B, fault)

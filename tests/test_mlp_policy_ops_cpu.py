"""CPU: the argument refusals of the MLP layer, LayerNorm parameter-gradient and policy std-head entry points.  Each is checked on
the host and returns SERL_ERR_INVALID with a message that names the entry point, before anything is enqueued, so no device is
needed; a call that got as far as a launch would fail here with SERL_ERR_CUDA instead."""
import re

import pytest

NUL, PTR = None, 256          # a null operand / a non-null one (never dereferenced: the call is refused first)
R, D, B, A = 26, 64, 13, 4


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as G
    G.build()
    from serl_b200 import _lib
    _lib.load()
    return _lib


def _refused(L, name, *args):
    before = L.launch_count()
    with pytest.raises(L.SerlError, match=rf"^{name} failed \({-1}\): {re.escape(name)}: "):
        L.call(name, *args)
    assert L.launch_count() == before


def _fwd(L, act, layer_norm, scale=PTR, bias=PTR, rows_per_group=B):
    _refused(L, "serl_layernorm_act_fwd", PTR, D, scale, bias, rows_per_group, D, PTR, D, PTR, PTR, R, D, 1e-6, act, layer_norm, NUL)


def _bwd(L, act, layer_norm, t=PTR, pre=PTR, scale=PTR, bias=PTR):
    _refused(L, "serl_layernorm_act_bwd", PTR, D, t, D, pre, D, PTR, PTR, scale, bias, B, D, PTR, PTR, R, D, act, layer_norm, NUL)


@pytest.mark.parametrize("act", [-1, 5, 99])
@pytest.mark.parametrize("layer_norm", [0, 1])
def test_layernorm_act_unknown_activation(L, act, layer_norm):
    _fwd(L, act, layer_norm)
    _bwd(L, act, layer_norm)


@pytest.mark.parametrize("act", range(5))
def test_layernorm_act_needs_scale_and_bias_with_layernorm(L, act):
    _fwd(L, act, 1, scale=NUL)
    _fwd(L, act, 1, bias=NUL)
    _fwd(L, act, 1, rows_per_group=0)
    _bwd(L, act, 1, scale=NUL)
    if act != L.ACT_TANH:               # tanh's derivative comes from its output t; the others recompute y = xhat * scale + bias
        _bwd(L, act, 1, bias=NUL)


@pytest.mark.parametrize("act", range(5))
def test_layernorm_act_bwd_needs_its_derivative_operand(L, act):
    if act == L.ACT_TANH:
        _bwd(L, act, 0, t=NUL)
        _bwd(L, act, 1, t=NUL)
    else:                               # without LayerNorm the pre-activation is read from `pre`
        _bwd(L, act, 0, pre=NUL)


def _std_args(L, std_param, ld_x, eps=PTR, deterministic=0):
    fwd = (PTR, PTR, ld_x, std_param, eps, 1e-5, 5.0, PTR, A, PTR, PTR, PTR, B, A, deterministic, NUL)
    loss = (PTR, PTR, PTR, PTR, A, PTR, A, PTR, PTR, ld_x, std_param, eps, 1e-5, 5.0, 1.0, PTR, PTR, PTR, 10, B, A, NUL)
    return fwd, loss


@pytest.mark.parametrize("std_param,ld_x", [(2, A), (2, 1), (2, -1), (0, 0), (1, 0), (0, -A), (3, A), (3, 0), (-1, A)])
def test_std_head_row_stride_and_parameterisation(L, std_param, ld_x):
    """The "uniform" head reads one (A,) leaf (ld_x == 0 exactly); "exp" / "softplus" read a (B, A) head output (ld_x > 0)."""
    fwd, loss = _std_args(L, std_param, ld_x)
    _refused(L, "serl_tanh_gaussian_fwd_std", *fwd)
    _refused(L, "serl_actor_loss_std", *loss)


@pytest.mark.parametrize("std_param", range(3))
def test_tanh_gaussian_fwd_std_needs_eps_unless_deterministic(L, std_param):
    fwd, _ = _std_args(L, std_param, 0 if std_param == L.STD_UNIFORM else A, eps=NUL)
    _refused(L, "serl_tanh_gaussian_fwd_std", *fwd)
    _refused(L, "serl_tanh_gaussian_fwd", PTR, PTR, NUL, 1e-5, 5.0, PTR, A, PTR, PTR, PTR, B, A, 0, NUL)


@pytest.mark.parametrize("rows_per_group,rows", [(13, 27), (13, 12), (256, 2559), (0, 26)])
def test_layernorm_param_grad_needs_whole_groups(L, rows_per_group, rows):
    _refused(L, "serl_layernorm_param_grad", PTR, PTR, PTR, PTR, rows_per_group, rows, D, NUL)

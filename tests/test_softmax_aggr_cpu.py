"""The SoftmaxAggregation mirror's constructor errors, parameters and repr match the reference's (basic.py:172-218),
and the softmax-aggregation wrappers check their operands before anything reaches the device."""
import pytest
import torch

from pytorch_geometric_b200 import ops
from pytorch_geometric_b200.nn import SoftmaxAggregation


def test_constructor_errors():
    with pytest.raises(ValueError, match="Cannot enable 'semi_grad' in 'SoftmaxAggregation' in case the temperature"):
        SoftmaxAggregation(learn=True, semi_grad=True)
    with pytest.raises(ValueError, match="Cannot set 'channels' greater than '1' in case 'SoftmaxAggregation' is not "
                                         "trainable"):
        SoftmaxAggregation(channels=4)


def test_parameters_reset_and_repr():
    agg = SoftmaxAggregation(t=0.25, learn=True, channels=3)
    assert isinstance(agg.t, torch.nn.Parameter) and agg.t.shape == (3, )
    assert torch.equal(agg.t.data, torch.full((3, ), 0.25))
    with torch.no_grad():
        agg.t.fill_(2.0)
    agg.reset_parameters()
    assert torch.equal(agg.t.data, torch.full((3, ), 0.25))
    assert list(agg.state_dict()) == ["t"]
    assert repr(agg) == "SoftmaxAggregation(learn=True)"
    fixed = SoftmaxAggregation(t=0.5)
    assert fixed.t == 0.5 and list(fixed.state_dict()) == [] and repr(fixed) == "SoftmaxAggregation(learn=False)"


def test_two_dimensional_input_with_channels():
    agg = SoftmaxAggregation(learn=True, channels=4)
    with pytest.raises(ValueError, match="two-dimensional inputs"):
        agg(torch.randn(3, 2, 4), torch.zeros(3, dtype=torch.long), dim_size=1)
    with pytest.raises(ValueError, match="first dimension"):
        agg.forward(torch.randn(4, 4), torch.zeros(4, dtype=torch.long), dim_size=1, dim=1)


def test_operand_checks():
    x = torch.randn(5, 8)
    a = torch.randn(7, 8)
    with pytest.raises(ValueError, match="message must be one of"):
        ops._softmax_aggr_args(x, None, None, "gelu", 7)
    with pytest.raises(ValueError, match="relu_eps message needs x"):
        ops._softmax_aggr_args(None, a, None, "relu_eps", 7)
    with pytest.raises(ValueError, match="exactly one of x and the edge rows"):
        ops._softmax_aggr_args(x, a, None, "identity", 7)
    with pytest.raises(ValueError, match="edge rows must have 6 rows"):
        ops._softmax_aggr_args(x, a, None, "relu_eps", 6)
    with pytest.raises(ValueError, match="t must be a contiguous float32 tensor of 1 or 8"):
        ops._softmax_aggr_args(x, a, torch.ones(3), "relu_eps", 7)
    with pytest.raises(ValueError, match="float32"):
        ops._softmax_aggr_args(x, a, torch.ones(8, dtype=torch.bfloat16), "relu_eps", 7)
    assert ops._softmax_aggr_args(x, a, torch.ones(8), "relu_eps", 7) == (8, 1, 2)
    assert ops._softmax_aggr_args(None, a, torch.ones(1), "identity", 7) == (8, 0, 1)
    assert ops._softmax_aggr_args(x, None, None, "identity", 7) == (8, 0, 0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        ops.softmax_aggr_csr(torch.zeros(3, dtype=torch.long), None, None, None, a, None, 2, 7)

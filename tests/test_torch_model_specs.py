"""torch.nn.Module predictors without a GPU: recognition, every refusal that needs no device, and the block planner of the
masked rows.  The module route itself runs in tests/test_gpu_torch_models.py."""
import numpy as np
import pytest
import torch
from sklearn.pipeline import Pipeline
from sklearn.preprocessing import StandardScaler

from distributedkernelshap_b200 import torch_models
from distributedkernelshap_b200.engine import GpuKernelExplainer
from distributedkernelshap_b200.explainers.kernel_shap import KernelShap
from distributedkernelshap_b200.torch_models import TorchModelSpec, is_torch_module, model_batch_rows, plan_blocks

BG = np.random.RandomState(0).randn(10, 3)


def _net(dtype=torch.float64):
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(3, 4), torch.nn.Tanh(), torch.nn.Linear(4, 2)).to(dtype).eval()


def test_recognises_modules_and_script_modules_only():
    net = _net()
    assert is_torch_module(net)
    assert is_torch_module(torch.jit.script(net))
    assert not is_torch_module(net.forward)
    assert not is_torch_module(lambda x: x)
    assert not is_torch_module(np.zeros(3))


def test_training_mode_is_refused_with_the_fix():
    with pytest.raises(ValueError, match=r"module\.eval\(\)"):
        TorchModelSpec(_net().train())
    with pytest.raises(ValueError, match="training mode"):
        GpuKernelExplainer(_net().train(), BG)
    net = _net().train()
    with pytest.raises(ValueError):
        TorchModelSpec(net)
    assert net.training                                   # the engine does not switch it for the user


def test_cpu_module_is_refused():
    with pytest.raises(ValueError, match="CUDA device"):
        TorchModelSpec(_net())
    with pytest.raises(ValueError, match="CUDA device"):
        GpuKernelExplainer(_net(), BG)


def test_mixed_dtypes_are_refused():
    net = _net()
    net[2].to(torch.float32)
    with pytest.raises(TypeError, match="mixes dtypes"):
        TorchModelSpec(net)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_precision_is_refused(dtype):
    with pytest.raises(TypeError, match="half and bfloat16"):
        TorchModelSpec(_net(dtype))


def test_module_without_floating_parameters_is_refused():
    with pytest.raises(TypeError, match="no floating parameter"):
        TorchModelSpec(torch.nn.Tanh().eval())


def test_distributed_opts_are_refused():
    with pytest.raises(NotImplementedError, match="distributed_opts"):
        KernelShap(_net(), distributed_opts={"n_cpus": 2})


def test_module_behind_a_pipeline_is_refused():
    pipe = Pipeline([("scale", StandardScaler()), ("net", _net())])
    with pytest.raises(TypeError, match="Pipeline"):
        GpuKernelExplainer(pipe, BG)


def test_numpy_callable_still_raises_type_error():
    with pytest.raises(TypeError):
        GpuKernelExplainer(lambda x: np.tanh(x).sum(axis=1), BG)


@pytest.mark.parametrize("value, N, want", [(None, 100, (1 << 20) // 100 * 100), (1, 100, 100), (250, 100, 200),
                                            (300, 100, 300), (7, 1, 7)])
def test_model_batch_rows_rounds_to_whole_coalitions(value, N, want):
    assert model_batch_rows(value, N) == want


def test_model_batch_rows_must_be_positive():
    with pytest.raises(ValueError):
        model_batch_rows(0, 10)


@pytest.mark.parametrize("coalitions, N, per", [(1, 100, 1), (7, 100, 1), (7, 100, 3), (7, 100, 7), (7, 100, 50),
                                                (1000, 13, 64), (0, 10, 2)])
def test_block_plan_covers_every_row_once_in_whole_coalitions(coalitions, N, per):
    total, batch = coalitions * N, per * N
    blocks = plan_blocks(total, N, batch)
    covered = np.zeros(total, dtype=int)
    for row0, rows in blocks:
        assert rows > 0 and rows <= batch
        assert row0 % N == 0 and rows % N == 0
        covered[row0:row0 + rows] += 1
    assert (covered == 1).all()
    assert len(blocks) == -(-coalitions // per)


def test_block_plan_refuses_partial_coalitions():
    with pytest.raises(ValueError):
        plan_blocks(250, 100, 100)
    with pytest.raises(ValueError):
        plan_blocks(200, 100, 150)


def test_limits_match_the_engine():
    from distributedkernelshap_b200 import _cabi
    assert torch_models.MAX_OUTPUTS == 8
    assert TorchModelSpec.act_code == _cabi.ACT_EXTERNAL

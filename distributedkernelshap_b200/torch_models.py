"""``torch.nn.Module`` predictors: recognition, the conditions the engine needs, and the block plan of the masked rows.

A module is a black box to the engine: it has no tables to fold a coalition into, so every coalition row of an instance is
materialised against every background row on the device (``dks_external_mask``), the module runs on those rows under
``torch.inference_mode()`` and the engine reduces its outputs over the background (``dks_external_reduce``) before the
link and the solve (DESIGN.md §5.0.19).  Nothing here calls the module on the CPU.
"""
import sys

import numpy as np

MAX_GROUPS = 64          # the ensemble tail and the coalition bits of one 64-bit word
MAX_OUTPUTS = 8          # DKS_ENS_MAX_OUT
DEFAULT_MODEL_BATCH_ROWS = 1 << 20


def _torch():
    import torch
    return torch


def is_torch_module(obj):
    """Whether ``obj`` is a ``torch.nn.Module`` (a ``torch.jit.ScriptModule`` included).  Without torch imported nothing
    can be one, so a NumPy-only caller does not pay for importing it."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(obj, torch.nn.Module)


def refuse_module_in_pipeline(model):
    """A ``Pipeline`` (or one of its bound methods) with a module among its steps: the engine would have to replay the
    steps in front of a black box, which it does not do."""
    owner = getattr(model, "__self__", model)
    steps = getattr(owner, "steps", None)
    if type(owner).__name__ == "Pipeline" and isinstance(steps, list):
        if any(is_torch_module(step) for _, step in steps):
            raise TypeError("a torch.nn.Module behind a scikit-learn Pipeline is not supported: put the preprocessing "
                            "inside the module and pass the module itself")


def model_batch_rows(value, N):
    """Masked rows per module call: ``value`` (default 2^20) rounded down to whole coalitions of ``N`` background rows,
    at least one coalition."""
    value = DEFAULT_MODEL_BATCH_ROWS if value is None else int(value)
    if value < 1:
        raise ValueError(f"model_batch_rows must be positive (got {value})")
    return max(N, value // N * N)


def plan_blocks(rows_total, N, batch_rows):
    """``[(row0, rows), ...]``: the masked rows ``0 .. rows_total - 1`` of an explain call in blocks of ``batch_rows``
    (a multiple of N), the last one shorter; every block non-empty and made of whole coalitions."""
    if rows_total % N or batch_rows % N or batch_rows < N:
        raise ValueError(f"rows_total={rows_total} and batch_rows={batch_rows} must be whole coalitions of N={N} rows")
    return [(r, min(batch_rows, rows_total - r)) for r in range(0, rows_total, batch_rows)]


class TorchModelSpec:
    """A module the engine explains by calling it between its launches.  Checked on construction: floating parameters
    (and floating buffers) on one CUDA device with one dtype, float32 or float64, and eval mode.  ``bind_background`` runs
    the module on the background, which fixes its width and outputs."""

    head = None
    activation = None
    maps = None
    R = 1
    act_code = 11                      # DKS_ACT_EXTERNAL

    def __init__(self, module):
        torch = _torch()
        params = [p for p in module.parameters()]
        floating = [t for t in params + list(module.buffers()) if t.is_floating_point()]
        if not any(p.is_floating_point() for p in params):
            raise TypeError("the module has no floating parameter: the engine takes the input dtype and device from its "
                            "parameters")
        dtypes = {t.dtype for t in floating}
        if len(dtypes) > 1:
            raise TypeError(f"the module mixes dtypes {sorted(map(str, dtypes))}: use one of float32 or float64")
        dtype = dtypes.pop()
        if dtype not in (torch.float32, torch.float64):
            raise TypeError(f"the module's parameters are {dtype}: float32 or float64 only (half and bfloat16 are not "
                            "supported)")
        if module.training:
            raise ValueError("the module is in training mode: call module.eval() before explaining it (dropout and "
                             "batch statistics would make its outputs depend on the batch)")
        devices = {t.device for t in floating}
        if len(devices) > 1:
            raise ValueError(f"the module's parameters are spread over several devices ({sorted(map(str, devices))}): "
                             "move it to one CUDA device")
        device = devices.pop()
        if device.type != "cuda":
            raise ValueError(f"the module is on {device}: the engine explains modules on a CUDA device (module.cuda())")
        self.module = module
        self.device = device.index if device.index is not None else torch.cuda.current_device()
        self.dtype = dtype
        self.dtype_code = 1 if dtype == torch.float64 else 0
        self.n_features = None
        self.n_outputs = None
        self.scalar_out = None

    def outputs(self, x):
        """The module on rows ``x`` [B, D] (on its device, its dtype) under ``inference_mode``: ``[B, C]`` float32 or
        float64, contiguous.  Raises for an output of the wrong rank, batch length, width or dtype (the first call, on
        the background, fixes C and whether the module returns ``[B]``)."""
        torch = _torch()
        with torch.inference_mode():
            y = self.module(x)
        if not isinstance(y, torch.Tensor):
            raise TypeError(f"the module returned {type(y).__name__}, not a tensor")
        B = x.shape[0]
        if y.dim() not in (1, 2) or y.shape[0] != B:
            raise ValueError(f"the module maps [{B}, {x.shape[1]}] to {list(y.shape)}: expected [{B}] or [{B}, C]")
        if y.device != x.device:
            raise ValueError(f"the module's output is on {y.device}, its input on {x.device}")
        if y.dtype not in (torch.float32, torch.float64):
            raise TypeError(f"the module's output is {y.dtype}: float32 or float64 only")
        scalar = y.dim() == 1
        y = y.reshape(B, -1)
        if self.n_outputs is None:
            if not 1 <= y.shape[1] <= MAX_OUTPUTS:
                raise ValueError(f"the module gives {y.shape[1]} outputs: 1 to {MAX_OUTPUTS} are supported")
            self.n_outputs, self.scalar_out = y.shape[1], scalar
        elif y.shape[1] != self.n_outputs or scalar != self.scalar_out:
            raise ValueError(f"the module gave {'[B]' if scalar else list(y.shape)} outputs on these rows, "
                             f"{'[B]' if self.scalar_out else [B, self.n_outputs]} on the background")
        return y.contiguous()

    def bind_background(self, bg):
        """The module's outputs on the background rows ``bg`` [N, P] (float64 NumPy), which fix its width P, its C
        outputs (1..8) and whether it returns ``[B]``."""
        torch = _torch()
        y = self.outputs(torch.as_tensor(bg, dtype=self.dtype, device=torch.device("cuda", self.device)))
        self.n_features = bg.shape[1]
        return y

    def predict(self, X):
        """The module's outputs on rows ``X`` (NumPy, any float) as float64 NumPy ``[n, C]``."""
        torch = _torch()
        x = torch.as_tensor(np.asarray(X, dtype=np.float64), dtype=self.dtype, device=torch.device("cuda", self.device))
        return self.outputs(x).double().cpu().numpy()

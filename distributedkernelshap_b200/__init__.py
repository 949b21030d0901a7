"""H100-native KernelSHAP engine behind the API of alexcoca/DistributedKernelShap.

Public surface (mirrors the reference's ``explainers`` package, reference file:line in each module):

    distributedkernelshap_b200.explainers.kernel_shap.KernelShap        fit / explain
    distributedkernelshap_b200.explainers.distributed.DistributedExplainer
    distributedkernelshap_b200.explainers.wrappers.KernelShapModel / BatchKernelShapModel
    distributedkernelshap_b200.engine.GpuKernelExplainer               the object in KernelShap._explainer

The numerical hot path is hand-written sm_90a CUDA in ``csrc/`` reached through the C ABI of
``include/dks.h`` (``libdks.so``) via ctypes.  There is no CPU fallback: without the library or a GPU the
engine raises.
"""

__version__ = "0.1.0"

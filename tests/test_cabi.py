"""The C-ABI library builds for sm_90a, loads, and exports every symbol include/dks.h declares.  No compute here."""
import ctypes
import os
import re

import pytest

from distributedkernelshap_b200 import _cabi, build

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(REPO, "include", "dks.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dks_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_declared_symbols():
    if build.find_nvcc() is None and not os.path.exists(build.LIB_PATH):
        pytest.skip("no nvcc and no prebuilt library")
    lib = _cabi.load()
    names = declared_symbols()
    assert len(names) >= 25
    for name in names:
        assert hasattr(lib, name), f"{name} declared in dks.h but not exported"
        assert name in _cabi.SIGNATURES, f"{name} has no ctypes signature"
    assert set(_cabi.SIGNATURES) == set(names)
    assert lib.dks_version() == 100


def test_sass_is_sm90a():
    if build.find_nvcc() is None:
        pytest.skip("no CUDA toolkit")
    import subprocess
    _cabi.load()
    out = subprocess.run(["cuobjdump", "-lelf", build.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_cpu_fallback_without_a_gpu():
    lib = _cabi.load()
    n = ctypes.c_int(-1)
    assert lib.dks_device_count(ctypes.byref(n)) == 0
    if n.value > 0:
        pytest.skip("a GPU is present")
    ctx = ctypes.c_void_p()
    rc = lib.dks_create(ctypes.byref(ctx), 0)
    assert rc == _cabi.DKS_ERR_CUDA and b"no CPU fallback" in lib.dks_last_error()
    from distributedkernelshap_b200.engine import GpuKernelExplainer
    from conftest import make_problem
    prob = make_problem()
    with pytest.raises(_cabi.DksError):
        GpuKernelExplainer(prob["clf"].predict_proba, prob["bg"], link="logit")


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(REPO, "distributedkernelshap_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(root, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{f} imports the oracle"
                assert "shap_kernel_oracle" not in src, f"{f} references the oracle module"


def _body_span(src, head):
    """(start, end) offsets of the first definition in src whose head (up to its opening brace) matches `head`."""
    m = re.search(head + r"\s*\{", src)
    assert m, f"{head} is not defined"
    depth, at = 0, m.end() - 1
    while True:
        depth += {"{": 1, "}": -1}.get(src[at], 0)
        if depth == 0:
            return m.start(), at
        at += 1


def test_only_the_buffer_owner_allocates():
    # every device and pinned-host allocation of the library goes through one allocate / free pair, which counts them
    # (dks_live_allocations); dks_host_alloc / dks_host_free hand page-locked memory to the caller
    csrc = os.path.join(REPO, "distributedkernelshap_b200", "csrc")
    allowed = {"dks_common.cuh": ("mem_alloc", "mem_free"), "dks.cu": ("dks_host_alloc", "dks_host_free")}
    calls = re.compile(r"\bcuda(Malloc\w*|Free\w*|HostAlloc|HostRegister)\b")
    for f in sorted(os.listdir(csrc)):
        src = open(os.path.join(csrc, f)).read()
        src = re.sub(r"//[^\n]*", "", re.sub(r"/\*.*?\*/", "", src, flags=re.S))
        spans = [_body_span(src, r"\b" + name + r"\([^;{]*\)") for name in allowed.get(f, ())]
        for m in calls.finditer(src):
            line = src.count("\n", 0, m.start()) + 1
            assert any(a <= m.start() < b for a, b in spans), f"{f}:{line}: {m.group(0)} outside the buffer owner"
    common = open(os.path.join(csrc, "dks_common.cuh")).read()
    start, end = _body_span(common, r"\bstruct dks_ctx")
    assert not re.search(r"\bcap_\w+", common[start:end]), "dks_ctx keeps a capacity beside a buffer"

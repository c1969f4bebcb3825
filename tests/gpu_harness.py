"""The fixtures the GPU test modules share: import them into a module's namespace with
`from gpu_harness import cg, kernel_family, FAMILIES` and pytest finds them there."""
import pytest

FAMILIES = ["jit", "jit_always", "aot", "general"]


@pytest.fixture(scope="module")
def cg():
    """the library, built for sm_90a, with device 0 initialised: the columnar module"""
    import torch
    assert torch.cuda.is_available(), "these tests need an H100"
    from citus_b200 import build
    build.build()
    from citus_b200 import columnar
    columnar.init(0)
    return columnar


@pytest.fixture
def kernel_family(cg):
    """runs a test body once per kernel family through the same C-ABI calls: kernel_family(name), name in FAMILIES"""
    def use(name):
        cg.set_option("jit", {"jit": 1, "jit_always": 2, "aot": 0, "general": 0}[name])
        cg.set_option("force_general", 1 if name == "general" else 0)
    yield use
    cg.set_option("jit", 1)
    cg.set_option("force_general", 0)

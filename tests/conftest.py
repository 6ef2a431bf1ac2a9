import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def oracle_lib():
    import oracle

    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def cuda_lib():
    """The product library; GPU tests fail loudly if it is missing or no GPU is visible."""
    import torch

    from newton_b200 import _lib

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return _lib.lib()


@pytest.fixture
def host_copies(oracle_lib, monkeypatch):
    """Lets CPU tests drive ``ArticulationView.set_*`` / index-gathers end to end: the one method that launches the CUDA copy
    kernels is replaced by ``orc_view_copy_product_host``, which executes the SAME index arithmetic (csrc/nb2_selection.cuh,
    host+device) word by word on the host.  Everything above it - selectors, layouts, the ``nb2_view_layout`` the product fills,
    value / mask handling - is the product code under test.  Test infrastructure only: the product has no CPU path."""
    import ctypes as C

    from newton_b200.selection import ArticulationView

    def launch(self, attrib, abi_layout, values, mask, gather):
        assert attrib.is_contiguous() and values.is_contiguous() and not attrib.is_cuda
        oracle_lib.lib().orc_view_copy_product_host(
            C.c_void_p(attrib.data_ptr()), C.byref(abi_layout), C.c_void_p(values.data_ptr()),
            C.c_void_p(None if mask is None else mask.data_ptr()), C.c_int(0 if mask is None else mask.dim()),
            C.c_int(1 if gather else 0), C.c_int(0))

    monkeypatch.setattr(ArticulationView, "_launch_copy", launch)
    return launch

import ctypes
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_package():
    name = "web_audio_api_rs_b200"
    if name in sys.modules:
        return sys.modules[name]
    pkg_dir = os.path.join(ROOT, "web-audio-api-rs_b200")
    spec = importlib.util.spec_from_file_location(name, os.path.join(pkg_dir, "__init__.py"),
                                                  submodule_search_locations=[pkg_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="session")
def pkg():
    return load_package()


@pytest.fixture(scope="session")
def oracle(pkg):
    """The CPU oracle (test infrastructure): built from oracle/ on first use."""
    so = os.path.join(ROOT, "oracle", "_build", "liboracle.so")
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-j8"], stdout=subprocess.DEVNULL)
    api = pkg.Api(ctypes.CDLL(so), "wao_")
    return pkg.context.Backend(api)


@pytest.fixture(params=["oracle", "engine"])
def host_api(request, pkg, oracle):
    """Host-only entry points (no device work) that BOTH libraries export: the oracle's and the product's own host code
    (libwae_b200.so loads without a GPU).  Tests using it pin the product's control-side math on the CPU."""
    if request.param == "oracle":
        return oracle.api
    so = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.api()


@pytest.fixture(params=["oracle", "engine"])
def builder(request, pkg, oracle):
    """A backend for tests that only BUILD graphs (validation, ids, processing order): the oracle, and the product's own graph
    half with no engine attached (wae_graph_create(NULL, ...): host work, runs without a GPU; rendering it raises)."""
    if request.param == "oracle":
        return oracle
    so = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


@pytest.fixture(scope="session")
def engine(pkg, oracle):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    e = pkg.Engine(0)
    yield e
    e.close()

"""CPU-side checks of the C-ABI library and the host mirror: the .so loads, exports exactly what
include/fluid.h declares, fails loudly without a GPU, and the host logic (config, getResolution,
colours, dt clamp) follows the reference."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import webgl_fluid_simulation_b200 as pkg
from webgl_fluid_simulation_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    pkg.build()
    return pkg.lib()


def test_header_and_library_agree(L):
    hdr = open(os.path.join(ROOT, "include", "fluid.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(fluid_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for s in declared:
        assert hasattr(L, s), s
    assert L.fluid_abi_version() == 2


def test_no_loopback_transport_in_the_product(L):
    """The in-process halo transport of the slab tests (tests/slab_loopback.cu, FLUID_TEST_LOOPBACK) is compiled
    only into the test build: the product exports no loopback symbol and carries no loopback code."""
    out = subprocess.run(["nm", "-C", _lib.SO_PATH], capture_output=True, text=True, check=True).stdout
    assert "loopback" not in out.lower()
    assert not hasattr(L, "fluid_loopback_link")


def test_stat_tables_match_the_header_enum():
    """fluid_stat keys: the Python STAT table and the JS one name every FLUID_STAT_* of the header,
    with the same value (the JS keys are the camelCase form of the same names)."""
    hdr = open(os.path.join(ROOT, "include", "fluid.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    body = re.search(r"typedef enum fluid_stat_key \{(.*?)\} fluid_stat_key;", hdr, re.S).group(1)
    enum = {k.lower(): int(v) for k, v in re.findall(r"FLUID_STAT_([A-Z0-9_]+)\s*=\s*(\d+)", body)}
    assert len(enum) == body.count("=") and len(set(enum.values())) == len(enum), body
    assert {"cvd_stream_launches": 7, "gradient_stream_launches": 8}.items() <= enum.items()
    assert _lib.STAT == enum
    js = open(os.path.join(ROOT, "webgl_fluid_simulation_b200", "js", "fluid-sim.js")).read()
    table = re.search(r"const STAT = \{(.*?)\};", js, re.S).group(1)
    js_stat = {k: int(v) for k, v in re.findall(r"(\w+)\s*:\s*(\d+)", table)}
    camel = {re.sub(r"_([a-z0-9])", lambda m: m.group(1).upper(), k).replace("P2p", "P2P"): v for k, v in enum.items()}
    assert js_stat == camel


def test_no_torch_types_in_the_abi():
    hdr = open(os.path.join(ROOT, "include", "fluid.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)      # signatures only, not the prose
    assert "torch" not in hdr.lower() and "at::" not in hdr and "#include <cuda" not in hdr


def test_config_defaults_match_reference(L):
    c = _lib.Config()
    L.fluid_config_default(C.byref(c))
    assert (c.sim_w, c.dye_w, c.pressure_iterations) == (128, 1024, 20)          # S:60-61, S:66
    assert np.float32(c.density_dissipation) == 1 and np.float32(c.velocity_dissipation) == np.float32(0.2)
    assert np.float32(c.pressure) == np.float32(0.8) and c.curl == 30 and c.splat_radius == 0.25
    d = pkg.default_config()
    assert d["SPLAT_FORCE"] == 6000 and d["PAUSED"] is False


@pytest.mark.parametrize("res,cw,ch,exp", [(128, 1024, 1024, (128, 128)), (128, 1920, 1080, (228, 128)),
                                           (128, 1080, 1920, (128, 228)), (1024, 800, 600, (1365, 1024))])
def test_get_resolution(res, cw, ch, exp):
    r = pkg.getResolution(res, cw, ch)                                           # S:1612-1624
    assert (r["width"], r["height"]) == exp


def test_create_fails_loudly_without_gpu(L):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(pkg.FluidError) as e:
        pkg.FluidSimulation({"SIM_RESOLUTION": 32, "DYE_RESOLUTION": 32})
    assert e.value.code == -2 and "no CPU path" in str(e.value)


def test_product_never_imports_the_oracle():
    """The product may MENTION the oracle in prose; it must never import, link, load or call it."""
    pk = os.path.join(ROOT, "webgl_fluid_simulation_b200")
    bad = re.compile(r"(from|import)\s+oracle|oracle\.\w+\(|\boracle_\w+\s*\(|fluid_oracle|oracle/")
    for dp, _, fs in os.walk(pk):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".c", ".h", ".js", "Makefile")):
                src = open(os.path.join(dp, f), errors="ignore").read()
                assert not bad.search(src), os.path.join(dp, f)


def test_hsv_and_wrap():
    assert pkg.HSVtoRGB(0.0, 1, 1) == {"r": 1, "g": 0, "b": 0}                     # S:1573-1597
    c = pkg.HSVtoRGB(1 / 3, 1, 1)
    assert abs(c["g"] - 1) < 1e-12 and c["r"] < 1e-9
    assert pkg.wrap(1.25, 0, 1) == 0.25 and pkg.wrap(5, 2, 2) == 2                # S:1599-1603

"""Live re-derivation of the committed golden fixtures from the UNMODIFIED reference, whenever its checkout is present
(SUPIR_REFERENCE_ROOT; elsewhere this file skips): the cheap generators of tests/golden/make_golden.py
are re-run into a scratch directory and must reproduce the committed files bit for bit. Together with
tests/test_oracle_vs_golden.py (oracle == fixtures) this pins oracle == reference without trusting a stale fixture."""
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import ref_stubs  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_stubs.reference_available(), reason="the reference checkout is not present")
G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def regen(tmp_path_factory):
    mg = importlib.import_module("make_golden")
    out = tmp_path_factory.mktemp("golden_live")
    saved = mg.HERE
    mg.HERE = str(out)
    try:
        mg.gen_bookkeeping()
        mg.gen_zero_modules()
        mg.gen_glvcontrol_tiny()
        mg.gen_sampler()
        mg.gen_colorfix()
        mg.gen_conditioner()
        mg.gen_vae_fast()
        mg.gen_util()
        mg.gen_options()
        mg.gen_prepared_conditioner()
    finally:
        mg.HERE = saved
    return str(out)


def _same_npz(a, b):
    fa, fb = np.load(a), np.load(b)
    assert sorted(fa.files) == sorted(fb.files)
    for k in fa.files:
        x, y = fa[k], fb[k]
        assert x.shape == y.shape and x.dtype == y.dtype, k
        assert x.tobytes() == y.tobytes(), f"{os.path.basename(a)}:{k} differs from the committed fixture"


def test_bookkeeping_and_weights_regenerate_bit_identically(regen):
    with open(os.path.join(regen, "bookkeeping.json")) as f, open(os.path.join(G, "bookkeeping.json")) as g:
        assert f.read() == g.read()
    _same_npz(os.path.join(regen, "gaussian_weights.npz"), os.path.join(G, "gaussian_weights.npz"))


@pytest.mark.parametrize("name", ["zero_modules.npz", "glvcontrol_tiny.npz", "sampler_toy.npz", "colorfix.npz", "conditioner.npz", "vae_tiny_fast.npz", "prepared_conditioner.npz"])
def test_tensor_fixtures_regenerate_bit_identically(regen, name):
    _same_npz(os.path.join(regen, name), os.path.join(G, name))


def test_util_fixture_and_options_regenerate_identically(regen):
    with open(os.path.join(regen, "util_reference.json")) as f, open(os.path.join(G, "util_reference.json")) as g:
        assert f.read() == g.read()
    for name in sorted(os.listdir(os.path.join(G, "options"))):
        with open(os.path.join(regen, "options", name), "rb") as f, open(os.path.join(G, "options", name), "rb") as g:
            assert f.read() == g.read(), name

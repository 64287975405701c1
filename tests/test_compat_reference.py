"""compat.install() makes the reference's own factory resolve the hot-path targets to this package's classes, and the live
reference still agrees with the committed fixtures (both when the reference checkout is present); the reference's run
configurations (copied unedited to tests/golden/options/) instantiate through this package's factory, and PreparedConditioner
reproduces the reference class's recorded outputs."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import ref_stubs  # noqa: E402

needs_reference = pytest.mark.skipif(not ref_stubs.reference_available(), reason="the reference checkout is not present")


@needs_reference
def test_install_rebinds_reference_targets():
    ns = ref_stubs.import_reference()
    import sgm.util as sgm_util
    import supir_b200.compat as compat
    saved = {}
    import importlib
    for modname, attrs in compat.PATCHES.items():
        try:
            mod = importlib.import_module(modname)
        except Exception:
            continue
        for a in attrs:
            saved[(modname, a)] = getattr(mod, a, None)
    try:
        done = compat.install(strict=False)
        assert ("sgm.modules.diffusionmodules.sampling", "TiledRestoreEDMSampler") in done
        assert ("SUPIR.modules.SUPIR_v0", "LightGLVUNet") in done
        smp = sgm_util.instantiate_from_config({
            "target": "sgm.modules.diffusionmodules.sampling.TiledRestoreEDMSampler",
            "params": {"num_steps": 5, "restore_cfg": 4.0, "s_churn": 0, "s_noise": 1.003, "tile_size": 128, "tile_stride": 64, "device": "cpu",
                       "discretization_config": {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"},
                       "guider_config": {"target": "sgm.modules.diffusionmodules.guiders.LinearCFG", "params": {"scale": 7.5, "scale_min": 4.0}}}})
        assert type(smp).__module__ == "supir_b200.sampling" and type(smp.guider).__module__ == "supir_b200.guiders"
        cls = sgm_util.get_obj_from_str("SUPIR.modules.SUPIR_v0.GLVControl")
        assert cls.__module__ == "supir_b200.nets"
        assert sgm_util.get_obj_from_str("sgm.modules.diffusionmodules.wrappers.ControlWrapper").__module__ == "supir_b200.wrappers"
    finally:
        for (modname, a), v in saved.items():
            if v is not None:
                setattr(importlib.import_module(modname), a, v)


@needs_reference
def test_install_conditioner_is_opt_in_and_resolves_through_the_reference_factory():
    ref_stubs.import_reference()
    import importlib
    import sgm.util as sgm_util
    import supir_b200.compat as compat
    E = importlib.import_module("sgm.modules.encoders.modules")
    saved = {}
    for modname, attrs in dict(compat.PATCHES, **compat.CONDITIONER_PATCHES).items():      # install() rebinds all of these
        try:
            m = importlib.import_module(modname)
        except Exception:
            continue
        saved.update({(m, a): getattr(m, a) for a in attrs if hasattr(m, a)})
    try:
        compat.install(strict=False)
        assert E.FrozenCLIPEmbedder.__module__ == "sgm.modules.encoders.modules"          # untouched by default
        compat.install(strict=False, conditioner=True)
        cls = sgm_util.get_obj_from_str("sgm.modules.GeneralConditionerWithControl")
        assert cls.__module__ == "supir_b200.conditioner"
        assert sgm_util.get_obj_from_str("sgm.modules.encoders.modules.FrozenOpenCLIPEmbedder2").__module__ == "supir_b200.conditioner"
    finally:
        for (m, a), v in saved.items():
            setattr(m, a, v)


@needs_reference
def test_reference_still_matches_bookkeeping_fixture():
    import json
    ns = ref_stubs.import_reference()
    with open(os.path.join(os.path.dirname(__file__), "golden", "bookkeeping.json")) as f:
        book = json.load(f)
    for case in book["sliding_windows"]:
        assert [list(c) for c in ns.sampling._sliding_windows(*case["args"])] == case["windows"]


def test_every_reference_yaml_instantiates_through_this_packages_factory():
    """The reference's options/SUPIR_v0.yaml, SUPIR_v0_tiled.yaml and SUPIR_v0_Juggernautv9_lightning.yaml, unedited: every `target:` string of the
    model section — engine, wrapper, denoiser, both networks, VAE, sampler + guider, the conditioner with both text towers at
    full size — resolves to this package's classes (built on the meta device: 4.8 B parameters cost nothing)."""
    import glob
    import torch
    from supir_b200.config import instantiate_from_config, load_yaml
    paths = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "options", "*.yaml")))
    assert len(paths) >= 3
    samplers = set()
    for path in paths:
        cfg = load_yaml(path, attr_access=True)
        with torch.device("meta"):
            m = instantiate_from_config(cfg.model)
        mods = {type(x).__module__ for x in (m, m.model, m.model.diffusion_model, m.model.control_model, m.denoiser, m.sampler, m.sampler.guider,
                                             m.first_stage_model, m.conditioner, *m.conditioner.embedders)}
        assert all(x.startswith("supir_b200.") for x in mods), (path, mods)
        keys = m.state_dict().keys()
        assert sum(k.startswith("conditioner.embedders.0.transformer.text_model.encoder.layers.") for k in keys) == 12 * 16
        assert sum(k.startswith("conditioner.embedders.1.model.transformer.resblocks.") for k in keys) == 32 * 12
        assert sum(p.numel() for p in m.model.parameters()) > 3.8e9
        assert cfg.SDXL_CKPT and cfg.SUPIR_CKPT_Q
        samplers.add(type(m.sampler).__name__)
    assert samplers == {"RestoreEDMSampler", "TiledRestoreEDMSampler", "RestoreDPMPP2MSampler"}


def test_prepared_conditioner_matches_the_reference_class(tmp_path):
    """sgm.modules.PreparedConditioner (modules.py:246-290): conditions loaded from .pth files and repeated to the batch,
    with and without an unconditional file, against what the reference's own class returns on the same inputs (recorded in
    tests/golden/prepared_conditioner.npz by tests/golden/make_golden.py): same tensors, same key order, same state_dict keys."""
    import json
    import numpy as np
    import torch
    from supir_b200.config import instantiate_from_config
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "prepared_conditioner.npz"))
    keys = json.loads(str(z["keys"]))
    c = {k: torch.from_numpy(z["in_c_" + k]) for k in ("crossattn", "vector")}
    uc = {k: torch.from_numpy(z["in_uc_" + k]) for k in ("crossattn", "vector")}
    torch.save(c, tmp_path / "c.pth")
    torch.save(uc, tmp_path / "uc.pth")
    batch = {"control": torch.from_numpy(z["in_control"])}
    for case, un in (("with_uc", str(tmp_path / "uc.pth")), ("no_uc", None)):
        mine = instantiate_from_config({"target": "sgm.modules.PreparedConditioner", "params": {"cond_pth": str(tmp_path / "c.pth"), "un_cond_pth": un}})
        assert type(mine).__module__ == "supir_b200.conditioner"
        a, au = mine.get_unconditional_conditioning(batch)
        ref = keys[case]
        assert list(a) == ref["c"] and all(torch.equal(a[k], torch.from_numpy(z[f"{case}_c_{k}"])) for k in a)
        if ref["uc"] is None:
            assert au is None
        else:
            assert list(au) == ref["uc"] and all(torch.equal(au[k], torch.from_numpy(z[f"{case}_uc_{k}"])) for k in au)
        assert list(mine.state_dict()) == ref["state_dict"]

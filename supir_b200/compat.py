"""Drop-in installation into a checkout of the reference (Fanghua-Yu/SUPIR).

The reference resolves every hot-path class by dotted string through `sgm.util.instantiate_from_config`
(sgm/util.py:168-185) and `get_obj_from_str` (sgm/models/diffusion.py:50-53). `install()` imports the reference's own
modules and rebinds those names to this package's classes, so `test.py` / `gradio_demo_tiled.py` — which only touch the
object returned by `create_SUPIR_model` — run unchanged on the H100 backend:

    python -c "import supir_b200.compat as c; c.install(); import runpy; runpy.run_path('test.py', run_name='__main__')" ...

SUPIRModel itself (orchestration, colour fix, checkpoint loading) stays the reference's, and so does the text conditioner
unless `install(conditioner=True)` also rebinds it to supir_b200.conditioner (same state_dict keys: the SDXL checkpoint's
`conditioner.embedders.*` weights load into it unchanged).
"""
import importlib

# reference module -> {attribute: replacement "module:attr" in this package}
PATCHES = {
    "sgm.modules.diffusionmodules.wrappers": {"ControlWrapper": "supir_b200.wrappers:ControlWrapper"},
    "sgm.modules.diffusionmodules.denoiser": {"DiscreteDenoiserWithControl": "supir_b200.denoiser:DiscreteDenoiserWithControl"},
    "sgm.modules.diffusionmodules.guiders": {"LinearCFG": "supir_b200.guiders:LinearCFG", "VanillaCFG": "supir_b200.guiders:VanillaCFG"},
    "sgm.modules.diffusionmodules.sampling": {
        "RestoreEDMSampler": "supir_b200.sampling:RestoreEDMSampler",
        "TiledRestoreEDMSampler": "supir_b200.sampling:TiledRestoreEDMSampler",
        "RestoreDPMPP2MSampler": "supir_b200.sampling:RestoreDPMPP2MSampler",
        "TiledRestoreDPMPP2MSampler": "supir_b200.sampling:TiledRestoreDPMPP2MSampler",
        "gaussian_weights": "supir_b200.sampling:gaussian_weights",
        "_sliding_windows": "supir_b200.sampling:_sliding_windows",
    },
    "SUPIR.modules.SUPIR_v0": {"GLVControl": "supir_b200.nets:GLVControl", "LightGLVUNet": "supir_b200.nets:LightGLVUNet",
                               "ZeroSFT": "supir_b200.nets:ZeroSFT", "ZeroCrossAttn": "supir_b200.nets:ZeroCrossAttn"},
    "sgm.models.autoencoder": {"AutoencoderKLInferenceWrapper": "supir_b200.vae:AutoencoderKLInferenceWrapper",
                               "AutoencoderKL": "supir_b200.vae:AutoencoderKL"},
    "SUPIR.utils.tilevae": {"VAEHook": "supir_b200.vae:VAEHook"},
    "SUPIR.models.SUPIR_model": {"VAEHook": "supir_b200.vae:VAEHook",
                                 "DiagonalGaussianDistribution": "supir_b200.vae:DiagonalGaussianDistribution",
                                 "wavelet_reconstruction": "supir_b200.colorfix:wavelet_reconstruction",
                                 "adaptive_instance_normalization": "supir_b200.colorfix:adaptive_instance_normalization"},
}


# opt-in (install(conditioner=True)): the text conditioner. Off by default: the reference's own classes tokenise with
# transformers / open_clip and run the towers through those packages; this package's towers take over the arithmetic only.
CONDITIONER_PATCHES = {
    "sgm.modules.encoders.modules": {
        "GeneralConditioner": "supir_b200.conditioner:GeneralConditioner",
        "GeneralConditionerWithControl": "supir_b200.conditioner:GeneralConditionerWithControl",
        "FrozenCLIPEmbedder": "supir_b200.conditioner:FrozenCLIPEmbedder",
        "FrozenOpenCLIPEmbedder2": "supir_b200.conditioner:FrozenOpenCLIPEmbedder2",
        "ConcatTimestepEmbedderND": "supir_b200.conditioner:ConcatTimestepEmbedderND",
        "PreparedConditioner": "supir_b200.conditioner:PreparedConditioner",
    },
    "sgm.modules": {"GeneralConditioner": "supir_b200.conditioner:GeneralConditioner",
                    "GeneralConditionerWithControl": "supir_b200.conditioner:GeneralConditionerWithControl"},
}


def _resolve(spec):
    mod, attr = spec.split(":")
    return getattr(importlib.import_module(mod), attr)


def install(strict=True, conditioner=False):
    """Rebind the reference's hot-path names (and, with conditioner=True, its text conditioner classes). Returns the list of
    (module, attribute) pairs that were patched."""
    done = []
    patches = dict(PATCHES, **CONDITIONER_PATCHES) if conditioner else PATCHES
    for modname, attrs in patches.items():
        try:
            mod = importlib.import_module(modname)
        except Exception:
            if strict:
                raise
            continue
        for attr, spec in attrs.items():
            setattr(mod, attr, _resolve(spec))
            done.append((modname, attr))
    return done

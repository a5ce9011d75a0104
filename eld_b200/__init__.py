"""eld_b200 - H100-native (sm_90a) implementation of ELD's synthetic-noise training path.

Host-side mirror of the reference seams (SURVEY 8b) over the C ABI in include/eld_b200.h:
    eld_b200.noise.NoiseModel        <- noise.NoiseModel            (reference noise.py:174)
    eld_b200.arch.unet               <- models.arch.unet             (models/arch/__init__.py:6)
    eld_b200.models.eld_model        <- models.eld_model / ELDModel  (models/ELD_model.py:352)
    eld_b200.engine.Engine           <- engine.Engine                (engine.py:10)
"""


def engine_available():
    """True once the U-Net training step is implemented behind the C ABI."""
    try:
        from . import _lib
        return hasattr(_lib.load(), 'eld_unet_train_step')
    except Exception:
        return False

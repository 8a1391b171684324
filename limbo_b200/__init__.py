"""limbo_b200 — H100-native (sm_90a) GP compute backend behind limbo::model::GP's interface.

Only what the hot path needs lives here: csrc/ (CUDA kernels + C ABI), the ctypes
binding, and the host-side mirror of the reference's model / kernel / mean / acqui /
opt policies for that path.  There is no CPU fallback."""
from . import acqui, kernel, mean, model, opt, params, synth  # noqa: F401
from .params import Params, defaults  # noqa: F401

__version__ = "0.1.0"

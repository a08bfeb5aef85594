"""deepspeech.pytorch_b200 — H100-native DeepSpeech2 train-step path (import as
`deepspeech_pytorch_b200`; the directory name carries a dot, so a one-file shim at the repo root
registers the package under that importable name)."""
from . import _lib
from ._lib import Ds2Error, get_lib
from .configs import (AdamConfig, BiDirectionalConfig, DataConfig, OptimConfig, SGDConfig, SpectConfig,
                      UniDirectionalConfig)
from .enums import DecoderType, RNNType, SpectrogramWindow
from .labels import LABELS


def set_precision(name: str):
    """'fp32' (FFMA everywhere), 'tf32' (wgmma tensor cores, TF32 operands for the dense GEMMs) or 'fp16' (the
    reference's `precision: 16`: fp16 operand copies for the recurrent stack's GEMMs, everything else as 'tf32').
    A `DeepSpeech(precision=16)` model selects 'fp16' by itself for its own calls."""
    code = {"fp32": _lib.PREC_FP32, "tf32": _lib.PREC_TF32, "fp16": _lib.PREC_F16}[name]
    _lib.check(get_lib().ds2_set_precision(code), "ds2_set_precision")


def get_precision() -> str:
    return {_lib.PREC_FP32: "fp32", _lib.PREC_TF32: "tf32", _lib.PREC_F16: "fp16"}[get_lib().ds2_get_precision()]


from . import ops  # noqa: E402
from .decoder import GreedyDecoder  # noqa: E402
from .model import DeepSpeech  # noqa: E402

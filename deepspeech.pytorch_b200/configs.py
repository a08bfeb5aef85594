"""Structured configs with the field names and defaults of the reference's
deepspeech_pytorch/configs/train_config.py:16-73, restated so that they are legal on
python >= 3.11 (the reference's mutable dataclass defaults at :41,:87-89 are not) and usable
without hydra/omegaconf installed."""
from dataclasses import dataclass, field

from .enums import DecoderType, RNNType, SpectrogramWindow


@dataclass
class SpectConfig:
    sample_rate: int = 16000
    window_size: float = .02
    window_stride: float = .01
    window: SpectrogramWindow = SpectrogramWindow.hamming


@dataclass
class BiDirectionalConfig:
    rnn_type: RNNType = RNNType.lstm
    hidden_size: int = 1024
    hidden_layers: int = 5


@dataclass
class UniDirectionalConfig(BiDirectionalConfig):
    lookahead_context: int = 20


@dataclass
class OptimConfig:
    learning_rate: float = 1.5e-4
    learning_anneal: float = 0.99
    weight_decay: float = 1e-5


@dataclass
class SGDConfig(OptimConfig):
    momentum: float = 0.9


@dataclass
class AdamConfig(OptimConfig):
    eps: float = 1e-8
    betas: tuple = (0.9, 0.999)


@dataclass
class AugmentationConfig:
    speed_volume_perturb: bool = False
    spec_augment: bool = False
    noise_dir: str = ''
    noise_prob: float = 0.4
    noise_min: float = 0.0
    noise_max: float = 0.5


@dataclass
class DataConfig:
    train_path: str = 'data/train_manifest.csv'
    val_path: str = 'data/val_manifest.csv'
    batch_size: int = 64
    num_workers: int = 4
    labels_path: str = 'labels.json'
    spect: SpectConfig = field(default_factory=SpectConfig)
    augmentation: AugmentationConfig = field(default_factory=AugmentationConfig)
    prepare_data_per_node: bool = True


@dataclass
class LMConfig:
    """deepspeech_pytorch/configs/inference_config.py:7-16 (the decoder settings of evaluation and transcription)"""
    decoder_type: DecoderType = DecoderType.greedy
    lm_path: str = ''           # ARPA n-gram model (.arpa or .arpa.gz) for beam search; KenLM binaries are refused
    top_paths: int = 1          # number of beams to return
    alpha: float = 0.0          # language-model weight (no effect without a language model)
    beta: float = 0.0           # word bonus (no effect without a language model)
    cutoff_top_n: int = 40      # characters with the highest probabilities considered per frame
    cutoff_prob: float = 1.0    # cumulative-probability pruning; 1.0 = none
    beam_width: int = 10
    lm_workers: int = 4         # ctcdecode's CPU worker count; ignored by the GPU decoder


@dataclass
class ModelConfig:
    """inference_config.py:19-23"""
    precision: int = 32         # 16: the recurrent stack's GEMMs and sweeps on fp16 operands (`set_precision('fp16')`)
    cuda: bool = True
    model_path: str = ''


@dataclass
class InferenceConfig:
    """inference_config.py:26-29"""
    lm: LMConfig = field(default_factory=LMConfig)
    model: ModelConfig = field(default_factory=ModelConfig)


@dataclass
class TranscribeConfig(InferenceConfig):
    """inference_config.py:32-36 (the settings of `run_transcribe` and `decode_results`)"""
    audio_path: str = ''        # WAV file to transcribe
    offsets: bool = False       # also return the frame offsets of the characters
    chunk_size_seconds: float = -1   # <= 0: the whole file in one forward


@dataclass
class EvalConfig(InferenceConfig):
    """inference_config.py:39-45 (the settings of `evaluate`); `verbose` and `save_output` are unused there too"""
    test_path: str = ''         # JSON manifest or directory of .wav files with transcripts under /txt/
    verbose: bool = True
    save_output: str = ''
    batch_size: int = 20
    num_workers: int = 4


@dataclass
class OptimizerConfig:
    """search_lm_params.py:15-31 (the settings of `search_lm_params`) plus `seed` and `output_path`.  `n_jobs` and
    the decoding use of `num_workers` have no effect on the GPU search; `num_workers` still sets the loader's file
    readers."""
    model_path: str = ''
    test_path: str = ''
    is_character_based: bool = True   # pick the best pair by CER (True) or WER (False)
    lm_path: str = ''
    beam_width: int = 10
    alpha_from: float = 0.0
    alpha_to: float = 3.0
    beta_from: float = 0.0
    beta_to: float = 1.0
    n_trials: int = 500
    n_jobs: int = 2
    precision: int = 16
    batch_size: int = 1
    num_workers: int = 1
    spect_cfg: SpectConfig = field(default_factory=SpectConfig)
    seed: int = 0               # seed of the trial draws (numpy.random.default_rng)
    output_path: str = ''       # where to write [[alpha, beta, wer, cer], ...] (select_lm_params.py's input)


def cfg_type(cfg):
    """OmegaConf.get_type(cfg) when omegaconf wraps the config, else type(cfg) (model.py:152,274,282)."""
    try:
        from omegaconf import OmegaConf  # optional
        t = OmegaConf.get_type(cfg)
        if t is not None:
            return t
    except Exception:
        pass
    return type(cfg)


def is_kind(cfg, *names):
    """dataclass-type dispatch by class name, so configs built from the reference's own
    deepspeech_pytorch.configs.train_config classes are accepted as well."""
    return any(c.__name__ in names for c in cfg_type(cfg).__mro__)

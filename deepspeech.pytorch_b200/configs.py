"""Structured configs with the field names and defaults of the reference's
deepspeech_pytorch/configs/train_config.py:16-73, restated so that they are legal on
python >= 3.11 (the reference's mutable dataclass defaults at :41,:87-89 are not) and usable
without hydra/omegaconf installed."""
from dataclasses import dataclass, field
from typing import Any, Optional

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
class AlignConfig:
    """the settings of `align_manifest` (no counterpart in the reference): forced alignment of a manifest's
    transcripts to its audio"""
    model: ModelConfig = field(default_factory=ModelConfig)
    manifest_path: str = ''     # JSON manifest or directory of .wav files with transcripts under /txt/
    output_path: str = ''       # JSON lines, one record per utterance in manifest order
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


@dataclass
class ModelCheckpointConf:
    """configs/lightning_config.py:6-22 (the settings of `FileCheckpointHandler`).  `every_n_train_steps`,
    `train_time_interval`, `save_on_train_epoch_end` and `filepath` must keep their defaults: `train` raises
    otherwise."""
    _target_: str = "pytorch_lightning.callbacks.ModelCheckpoint"
    filepath: Optional[str] = None
    monitor: Optional[str] = None
    verbose: bool = False
    save_last: Optional[bool] = None
    save_top_k: Optional[int] = 1
    save_weights_only: bool = False
    mode: str = "min"
    dirpath: Any = None
    filename: Optional[str] = None
    auto_insert_metric_name: bool = True
    every_n_train_steps: Optional[int] = None
    train_time_interval: Optional[str] = None
    every_n_epochs: Optional[int] = None
    save_on_train_epoch_end: Optional[bool] = None


@dataclass
class TrainerConf:
    """configs/lightning_config.py:25-78, the Lightning Trainer's arguments.  `train` honours max_epochs, min_epochs,
    precision, gradient_clip_val, check_val_every_n_epoch, limit_train_batches, limit_val_batches,
    log_every_n_steps, enable_checkpointing, default_root_dir and resume_from_checkpoint; it does not read
    accelerator, devices, strategy, num_nodes (the process count comes from torchrun), logger, enable_progress_bar,
    enable_model_summary, num_sanity_val_steps and benchmark; any other field away from its default raises."""
    _target_: str = "pytorch_lightning.trainer.Trainer"
    logger: Any = True
    enable_checkpointing: bool = True
    default_root_dir: Optional[str] = None
    gradient_clip_val: float = 0
    callbacks: Any = None
    num_nodes: int = 1
    num_processes: int = 1
    gpus: Any = None
    auto_select_gpus: bool = False
    tpu_cores: Any = None
    overfit_batches: Any = 0.0
    track_grad_norm: Any = -1
    check_val_every_n_epoch: int = 1
    fast_dev_run: Any = False
    accumulate_grad_batches: Any = 1
    max_epochs: int = 1000
    min_epochs: int = 1
    limit_train_batches: Any = 1.0
    limit_val_batches: Any = 1.0
    limit_test_batches: Any = 1.0
    val_check_interval: Any = 1.0
    log_every_n_steps: int = 50
    accelerator: Any = None
    sync_batchnorm: bool = False
    precision: int = 32
    weights_save_path: Optional[str] = None
    num_sanity_val_steps: int = 2
    resume_from_checkpoint: Any = None
    profiler: Any = None
    benchmark: bool = False
    deterministic: bool = False
    auto_lr_find: Any = False
    replace_sampler_ddp: bool = True
    detect_anomaly: bool = False
    auto_scale_batch_size: Any = False
    plugins: Any = None
    amp_backend: str = "native"
    amp_level: Any = None
    move_metrics_to_cpu: bool = False
    gradient_clip_algorithm: Optional[str] = None
    devices: Any = None
    ipus: Optional[int] = None
    enable_progress_bar: bool = True
    max_time: Optional[str] = None
    limit_predict_batches: float = 1.0
    strategy: Optional[str] = None
    enable_model_summary: bool = True
    reload_dataloaders_every_n_epochs: int = 0
    multiple_trainloader_mode: str = "max_size_cycle"


@dataclass
class DeepSpeechConfig:
    """configs/train_config.py:81-91 (the settings of `train`).  Without hydra the defaults list (adam, bidirectional,
    file checkpoint) becomes the field defaults.  As in the reference, the data loaders read `data.augmentation`;
    the top-level `augmentation` is carried but unused."""
    optim: Any = field(default_factory=AdamConfig)
    model: Any = field(default_factory=BiDirectionalConfig)
    checkpoint: ModelCheckpointConf = field(default_factory=ModelCheckpointConf)
    trainer: TrainerConf = field(default_factory=TrainerConf)
    data: DataConfig = field(default_factory=DataConfig)
    augmentation: AugmentationConfig = field(default_factory=AugmentationConfig)
    seed: int = 123456
    load_auto_checkpoint: bool = False


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

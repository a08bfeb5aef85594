"""Writes tests/golden/training/reference_training.json from the reference itself: the field defaults of its
`TrainerConf`, `ModelCheckpointConf` and `DeepSpeechConfig` (configs/lightning_config.py, configs/train_config.py) and
the bin orders its `DSRandomSampler` / `DSElasticDistributedSampler` (loader/data_loader.py:282-360) yield for several
dataset sizes, batch sizes, world sizes and epochs.  The reference's imports that do not bear on these (librosa, sox,
torchaudio, omegaconf, the spec_augment module) are satisfied by inert stand-ins; the code that runs is its own.

    python tools/make_training_golden.py --reference <deepspeech.pytorch checkout>"""
import argparse
import dataclasses
import enum
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "training", "reference_training.json")

# (dataset size, batch size) x epochs x world sizes: uneven last bins, bin counts not divisible by the world size
CASES = [(37, 8), (40, 8), (5, 2), (11, 4)]
EPOCHS = [0, 1, 2, 7]
WORLDS = [1, 2, 3]
NP_SEED = 1234


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _jsonable(v):
    if isinstance(v, enum.Enum):
        return v.name
    if isinstance(v, tuple):
        return list(v)
    return v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True)
    args = ap.parse_args()
    sys.path.insert(0, args.reference)
    _stub("omegaconf", MISSING="???")
    for name in ("librosa", "sox"):
        _stub(name)
    _stub("torchaudio", set_audio_backend=lambda *a, **k: None)
    _stub("deepspeech_pytorch.loader.spec_augment", spec_augment=None)
    # python >= 3.11 refuses the reference's dataclass-instance defaults (train_config.py:41,87-89) unless the
    # classes hash; hashing changes no default
    plain = dataclasses.dataclass
    dataclasses.dataclass = lambda cls=None, **kw: plain(cls, unsafe_hash=True, **kw) if cls is not None else \
        (lambda c: plain(c, unsafe_hash=True, **kw))
    try:
        from deepspeech_pytorch.configs import lightning_config as LC
        from deepspeech_pytorch.configs import train_config as TC
        from deepspeech_pytorch.loader.data_loader import DSElasticDistributedSampler, DSRandomSampler
    finally:
        dataclasses.dataclass = plain
    # torch >= 2.2's Sampler takes no `data_source` (data_loader.py:290 passes one); the base class keeps nothing
    torch.utils.data.Sampler.__init__ = lambda self, *a, **k: None

    def defaults(cls):
        out = {}
        for f in dataclasses.fields(cls):
            if f.default is not dataclasses.MISSING:
                v = f.default
            elif f.default_factory is not dataclasses.MISSING:
                v = f.default_factory()
            else:
                continue
            out[f.name] = None if dataclasses.is_dataclass(v) else _jsonable(v)
        return out

    golden = {"TrainerConf": defaults(LC.TrainerConf), "ModelCheckpointConf": defaults(LC.ModelCheckpointConf),
              "DeepSpeechConfig": {k: v for k, v in defaults(TC.DeepSpeechConfig).items()
                                   if k in ("seed", "load_auto_checkpoint")},
              "np_seed": NP_SEED, "samplers": []}
    for n, bs in CASES:
        ds = list(range(n))
        for world in WORLDS:
            np.random.seed(NP_SEED)
            if world == 1:
                samplers = [DSRandomSampler(ds, batch_size=bs)]
            else:
                samplers = [DSElasticDistributedSampler(ds, num_replicas=world, rank=r, batch_size=bs)
                            for r in range(world)]
            orders = []
            for epoch in EPOCHS:       # one sampler object per rank over all epochs: the in-place shuffles carry over
                per_rank = []
                for s in samplers:
                    s.set_epoch(epoch)
                    per_rank.append([list(map(int, b)) for b in s])
                orders.append(per_rank)
            golden["samplers"].append({"n": n, "batch_size": bs, "world": world, "epochs": EPOCHS,
                                       "orders": orders})
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(golden, f, indent=None, separators=(",", ":"))
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()

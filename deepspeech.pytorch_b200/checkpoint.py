"""The reference's checkpoint.py (`FileCheckpointHandler`, a Lightning `ModelCheckpoint`) without Lightning: which
checkpoint files a training run keeps at each epoch end, under which names, and the newest one to resume from.

The rules are Lightning's: file names from the `filename` template with `{epoch}`, `{step}` and the logged metrics
(`{wer}`, `{cer}`), `name=` inserted before each when `auto_insert_metric_name` is set, `-v1`, `-v2`, ... appended when
the name is taken; the `save_top_k` best by `monitor` under `mode` (without a monitor: the newest, or all with -1);
`last.ckpt` with `save_last`; every `every_n_epochs` epochs.  The handler only decides and names: the caller passes a
function that writes the checkpoint to a path."""
import os
import re
from pathlib import Path

from . import _lib

CHECKPOINT_JOIN_CHAR = "-"
CHECKPOINT_NAME_LAST = "last"
FILE_EXTENSION = ".ckpt"
STARTING_VERSION = 1


class FileCheckpointHandler:
    def __init__(self, cfg, default_root_dir=None):
        """cfg: ModelCheckpointConf.  `default_root_dir` (TrainerConf.default_root_dir, else the working directory)
        places the default `dirpath`, `<root>/lightning_logs/version_N/checkpoints`, with N the next free version;
        that directory is chosen at the first save."""
        if cfg.mode not in ("min", "max"):
            raise _lib.Ds2Error(f"checkpoint.mode: {cfg.mode!r} is not one of 'min', 'max'")
        self.save_top_k = 1 if cfg.save_top_k is None else int(cfg.save_top_k)
        if self.save_top_k < -1:
            raise _lib.Ds2Error(f"checkpoint.save_top_k: {cfg.save_top_k} must be >= -1")
        if cfg.monitor is None and self.save_top_k not in (-1, 0, 1):
            raise _lib.Ds2Error(f"checkpoint.save_top_k: {cfg.save_top_k} needs checkpoint.monitor; without a "
                                "monitor only -1, 0 and 1 are valid")
        self.every_n_epochs = 1 if cfg.every_n_epochs is None else int(cfg.every_n_epochs)
        if self.every_n_epochs < 0:
            raise _lib.Ds2Error(f"checkpoint.every_n_epochs: {cfg.every_n_epochs} must be >= 0")
        self.monitor, self.mode, self.verbose = cfg.monitor, cfg.mode, bool(cfg.verbose)
        self.save_last, self.save_weights_only = bool(cfg.save_last), bool(cfg.save_weights_only)
        self.filename, self.auto_insert_metric_name = cfg.filename, bool(cfg.auto_insert_metric_name)
        self.root = os.path.abspath(default_root_dir or os.getcwd())
        self.dirpath = None if cfg.dirpath is None else os.path.abspath(os.path.expanduser(str(cfg.dirpath)))
        self.best_k_models = {}
        self.kth_best_model_path = ""
        self.kth_value = float("inf") if self.mode == "min" else float("-inf")
        self.best_model_path = ""
        self.best_model_score = None
        self.current_score = None
        self.last_model_path = ""

    # ------------------------------------------------------------------ where
    def resolve_dirpath(self):
        """the checkpoint directory; the default one is fixed by the first call"""
        if self.dirpath is None:
            logs = os.path.join(self.root, "lightning_logs")
            versions = [int(d[len("version_"):]) for d in (os.listdir(logs) if os.path.isdir(logs) else [])
                        if d.startswith("version_") and d[len("version_"):].isdigit()]
            self.dirpath = os.path.join(logs, f"version_{max(versions) + 1 if versions else 0}", "checkpoints")
        return self.dirpath

    def find_latest_checkpoint(self):
        """checkpoint.py:34-46: the newest file (by ctime) under `dirpath` -- under `<root>/lightning_logs` while no
        dirpath is set -- or None"""
        where = Path(self.dirpath if self.dirpath is not None else os.path.join(self.root, "lightning_logs"))
        paths = [p for p in where.rglob('*') if p.is_file()] if where.is_dir() else []
        if not paths:
            return None
        paths.sort(key=os.path.getctime)
        return paths[-1]

    # ------------------------------------------------------------------ names
    def format_checkpoint_name(self, metrics, filename=None, ver=None):
        """Lightning's `_format_checkpoint_name`: '{epoch}-{step}' without a template; each '{name' of the template
        becomes 'name={name' with auto_insert_metric_name; a metric the run does not have formats as 0"""
        filename = filename if filename is not None else self.filename
        if not filename:
            filename = "{epoch}" + CHECKPOINT_JOIN_CHAR + "{step}"
        metrics = dict(metrics)
        for group in re.findall(r"(\{.*?)[:\}]", filename):
            name = group[1:]
            if self.auto_insert_metric_name:
                filename = filename.replace(group, name + "={" + name)
            filename = filename.replace(group, f"{{0[{name}]")
            metrics.setdefault(name, 0)
        filename = filename.format(metrics)
        if ver is not None:
            filename = CHECKPOINT_JOIN_CHAR.join((filename, f"v{ver}"))
        return os.path.join(self.resolve_dirpath(), filename + FILE_EXTENSION)

    def _free_name(self, metrics, del_filepath=None):
        path = self.format_checkpoint_name(metrics)
        ver = STARTING_VERSION
        while os.path.exists(path) and path != del_filepath:
            path = self.format_checkpoint_name(metrics, ver=ver)
            ver += 1
        return path

    # ------------------------------------------------------------------ when and which
    def on_epoch_end(self, epoch, step, metrics, save):
        """after epoch `epoch` (0-based) at global step `step`, with the logged `metrics` ({'wer': .., 'cer': ..});
        `save(path)` writes a checkpoint.  Returns the path of the top-k checkpoint written, else None."""
        if self.every_n_epochs < 1 or (epoch + 1) % self.every_n_epochs:
            return None
        cand = {"epoch": int(epoch), "step": int(step), **{k: float(v) for k, v in metrics.items()}}
        written = self._save_top_k(cand, save) if self.save_top_k else None
        if self.save_last:
            path = self.format_checkpoint_name(cand, filename=CHECKPOINT_NAME_LAST)
            save(path)
            if self.last_model_path and self.last_model_path != path and os.path.exists(self.last_model_path):
                os.remove(self.last_model_path)
            self.last_model_path = path
        return written

    def _save_top_k(self, cand, save):
        if self.monitor is None:
            path = self._free_name(cand)
            previous, self.best_model_path = self.best_model_path, path
            save(path)
            if self.save_top_k == 1 and previous and previous != path and os.path.exists(previous):
                os.remove(previous)
            return path
        if self.monitor not in cand:
            raise _lib.Ds2Error(f"checkpoint.monitor: {self.monitor!r} is not a logged metric; the run logs "
                                f"{sorted(cand)}")
        current = cand[self.monitor]
        if not self._is_top_k(current):
            if self.verbose:
                print(f"Epoch {cand['epoch']:d}, global step {cand['step']:d}: {self.monitor!r} was not in top "
                      f"{self.save_top_k}")
            return None
        k = len(self.best_k_models) + 1 if self.save_top_k == -1 else self.save_top_k
        del_filepath = None
        if len(self.best_k_models) == k and k > 0:
            del_filepath = self.kth_best_model_path
            self.best_k_models.pop(del_filepath)
        if current != current:   # nan is never better
            current = float("inf") if self.mode == "min" else float("-inf")
        path = self._free_name(cand, del_filepath)
        self.current_score = current
        self.best_k_models[path] = current
        if len(self.best_k_models) == k:
            worst = max if self.mode == "min" else min
            self.kth_best_model_path = worst(self.best_k_models, key=self.best_k_models.get)
            self.kth_value = self.best_k_models[self.kth_best_model_path]
        best = min if self.mode == "min" else max
        self.best_model_path = best(self.best_k_models, key=self.best_k_models.get)
        self.best_model_score = self.best_k_models[self.best_model_path]
        if self.verbose:
            print(f"Epoch {cand['epoch']:d}, global step {cand['step']:d}: {self.monitor!r} reached {current:0.5f} "
                  f"(best {self.best_model_score:0.5f}), saving model to {path!r} as top {k}")
        save(path)
        if del_filepath is not None and path != del_filepath and os.path.exists(del_filepath):
            os.remove(del_filepath)
        return path

    def _is_top_k(self, current):
        if self.save_top_k == -1 or len(self.best_k_models) < self.save_top_k:
            return True
        return current < self.kth_value if self.mode == "min" else current > self.kth_value

    # ------------------------------------------------------------------ resume
    def state_dict(self):
        return {"monitor": self.monitor, "best_model_score": self.best_model_score,
                "best_model_path": self.best_model_path, "current_score": self.current_score,
                "dirpath": self.dirpath, "best_k_models": dict(self.best_k_models),
                "kth_best_model_path": self.kth_best_model_path, "kth_value": self.kth_value,
                "last_model_path": self.last_model_path}

    def load_state_dict(self, sd):
        """as Lightning does: the best-k bookkeeping only when it describes this handler's directory.  A handler
        without a `dirpath` of its own continues in the checkpoint's directory."""
        if self.dirpath is None or sd.get("dirpath") == self.dirpath:
            self.dirpath = sd.get("dirpath", self.dirpath)
            self.best_model_score = sd["best_model_score"]
            self.kth_best_model_path = sd["kth_best_model_path"]
            self.kth_value = sd["kth_value"]
            self.best_k_models = dict(sd["best_k_models"])
            self.last_model_path = sd["last_model_path"]
            self.current_score = sd.get("current_score")
        self.best_model_path = sd["best_model_path"]

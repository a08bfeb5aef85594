"""Language-model weight search, the reference's search_lm_params.py, on the GPU.

The reference reruns `run_evaluation` over the whole test set once per (alpha, beta) trial.  The acoustic outputs do
not depend on the pair, so `LMParamSearch` runs the model once, keeps the probabilities and the references on the
device, and evaluates many pairs per launch: `ds2_beam_decode_lm_grid` (one beam search per (utterance, pair)) and
`ds2_error_counts` (the WER / CER edit counts).  Only the final (K, 4) counts are copied to the host.

Differences from the reference: the trials are drawn uniformly and independently with `numpy.random.default_rng(seed)`
-- optuna's adaptive TPE sampler is not reproduced (optuna is not a dependency); `n_jobs` and the decoding use of
`num_workers` are ignored, as `BeamCTCDecoder` ignores `num_processes`."""
import json

import numpy as np
import torch

from . import _lib
from .decoder import BeamCTCDecoder, GreedyDecoder
from .evaluation import (AudioDataLoader, SpectrogramDataset, _space_of, error_counts, load_model, model_forward,
                         rates)

__all__ = ["LMParamSearch", "sample_pairs", "best_result", "write_results", "search_lm_params"]


class LMParamSearch:
    """`LMParamSearch(test_loader, model, decoder)`: runs `model` once over the loader (validation.py:158-161) and
    keeps, per utterance, the output probabilities, the output length and the reference labels on the device.
    `decoder` is a BeamCTCDecoder with a language model; its width and cutoffs are used, its alpha / beta are not.
    `evaluate(pairs)` -> [(alpha, beta, wer, cer)] in the order given, each equal to `run_evaluation` with
    `BeamCTCDecoder(lm_path, alpha, beta)` on the same loader.

    The utterances are sorted by output length (longest first) and split into groups of `group_size`; a group is
    padded only to its own longest utterance.  Each launch decodes one group for a chunk of pairs, as many pairs as
    keep its (pairs, group, T) label buffer under `label_bytes`, so that a launch has many items (group x pairs) per
    resident CTA."""

    def __init__(self, test_loader, model, decoder, target_decoder=None, precision=16, group_size=256,
                 label_bytes=256 << 20):
        if not isinstance(decoder, BeamCTCDecoder) or decoder.lm is None:
            raise _lib.Ds2Error("LMParamSearch: decoder must be a BeamCTCDecoder with a language model (lm_path)")
        self.decoder = decoder
        self.target_decoder = target_decoder or GreedyDecoder(decoder.labels, blank_index=decoder.blank_index)
        self.blank = self.target_decoder.blank_index
        self.space = _space_of(self.target_decoder.labels)
        self.label_bytes = int(label_bytes)
        utts = []                                    # (length, probs row, reference labels)
        model.eval()
        with torch.no_grad():
            for inputs, targets, input_percentages, target_sizes in test_loader:
                input_sizes = input_percentages.mul_(int(inputs.size(3))).int()
                out, output_sizes, _ = model_forward(model, inputs.cuda() if not inputs.is_cuda else inputs,
                                                     input_sizes, precision)
                out = out.float()
                tg = torch.as_tensor(targets).cpu()
                off = 0
                for b, (n, s) in enumerate(zip(torch.as_tensor(output_sizes).tolist(),
                                               torch.as_tensor(target_sizes).tolist())):
                    utts.append((int(n), out[b, :max(int(n), 1)].clone(), tg[off:off + s].clone()))
                    off += s
        if not utts:
            raise _lib.Ds2Error("LMParamSearch: the loader yielded no utterances")
        self.device = utts[0][1].device
        order = sorted(range(len(utts)), key=lambda i: utts[i][0], reverse=True)      # stable
        self.groups = []
        for g0 in range(0, len(order), max(1, int(group_size))):
            idx = order[g0:g0 + max(1, int(group_size))]
            T = max(utts[i][1].shape[0] for i in idx)
            Cn = utts[idx[0]][1].shape[1]
            probs = torch.zeros(len(idx), T, Cn, dtype=torch.float32, device=self.device)
            for r, i in enumerate(idx):
                probs[r, :utts[i][1].shape[0]] = utts[i][1]
            sizes = torch.tensor([utts[i][0] for i in idx], dtype=torch.int32)
            tsz = torch.tensor([utts[i][2].numel() for i in idx], dtype=torch.int32)
            tg = torch.cat([utts[i][2] for i in idx]).to(torch.int64)
            self.groups.append((probs, sizes.to(self.device), tg.to(self.device), tsz))
        del utts
        self.n_utterances = len(order)
        self.device_bytes = sum(p.numel() * 4 + s.numel() * 4 + t.numel() * 8 for p, s, t, _ in self.groups)

    def evaluate(self, pairs):
        """[(alpha, beta)] -> [(alpha, beta, wer, cer)], in the order given"""
        pr = np.asarray(pairs, dtype=np.float64).reshape(-1, 2)
        K = pr.shape[0]
        if K < 1:
            raise _lib.Ds2Error("LMParamSearch.evaluate: no (alpha, beta) pairs")
        if not np.all(np.isfinite(pr)):
            raise _lib.Ds2Error("LMParamSearch.evaluate: alpha and beta must be finite")
        counts = torch.zeros(K, 4, dtype=torch.int64, device=self.device)
        for probs, sizes, targets, tsz in self.groups:
            G, T, _ = probs.shape
            kc = max(1, min(K, self.label_bytes // max(1, G * T * 4)))
            for k0 in range(0, K, kc):
                k1 = min(K, k0 + kc)
                labels, lengths = self.decoder.decode_best_grid(probs, sizes, pr[k0:k1])
                error_counts(labels, lengths, targets, tsz, self.blank, self.space, pair_counts=counts[k0:k1],
                             rows=False)
        return [(float(a), float(b)) + rates(c) for (a, b), c in zip(pr.tolist(), counts.cpu().tolist())]


def sample_pairs(cfg):
    """n_trials pairs: alpha ~ U[alpha_from, alpha_to), then beta ~ U[beta_from, beta_to), each an array of
    n_trials draws from numpy.random.default_rng(cfg.seed)"""
    rng = np.random.default_rng(cfg.seed)
    a = rng.uniform(cfg.alpha_from, cfg.alpha_to, size=cfg.n_trials)
    b = rng.uniform(cfg.beta_from, cfg.beta_to, size=cfg.n_trials)
    return [(float(x), float(y)) for x, y in zip(a, b)]


def best_result(results, is_character_based):
    """the (alpha, beta, wer, cer) with the lowest CER (is_character_based) or WER; the earliest on a tie"""
    col = 3 if is_character_based else 2
    return min(results, key=lambda r: r[col])        # min keeps the first of equal keys


def write_results(path, results):
    """[[alpha, beta, wer, cer], ...]: the JSON select_lm_params.py reads"""
    with open(path, "w") as f:
        json.dump([[float(x) for x in r] for r in results], f)


def search_lm_params(cfg):
    """search_lm_params.py:101-115 (cfg: OptimizerConfig): evaluates cfg.n_trials sampled pairs, prints the reference's
    "Best Params" text, writes the results to cfg.output_path if set, and returns them"""
    device = torch.device("cuda")
    model = load_model(device, cfg.model_path)
    labels = model.labels
    decoder = BeamCTCDecoder(labels=labels, lm_path=cfg.lm_path, beam_width=cfg.beam_width,
                             num_processes=cfg.num_workers, blank_index=labels.index('_'))
    target_decoder = GreedyDecoder(labels=labels, blank_index=labels.index('_'))
    test_dataset = SpectrogramDataset(audio_conf=cfg.spect_cfg, input_path=cfg.test_path, labels=labels,
                                      normalize=True)
    test_loader = AudioDataLoader(test_dataset, batch_size=cfg.batch_size, num_workers=cfg.num_workers)
    search = LMParamSearch(test_loader, model, decoder, target_decoder, precision=cfg.precision)
    print(f"LMParamSearch: {search.n_utterances} utterances, {search.device_bytes} bytes kept on the device")
    results = search.evaluate(sample_pairs(cfg))
    alpha, beta, wer, cer = best_result(results, cfg.is_character_based)
    print(f"Best Params\n"
          f"alpha: {alpha}\n"
          f"beta: {beta}\n"
          f"{'cer' if cfg.is_character_based else 'wer'}: {cer if cfg.is_character_based else wer}")
    if cfg.output_path:
        write_results(cfg.output_path, results)
    return results

"""Data-loader builders (reference ``fms_fsdp/utils/dataloader_utils.py:17-163``).

``get_dummy_loader`` -- steady synthetic stream used for all benchmarking (``use_dummy_dataset``);
``get_data_loader`` -- the production 8-stage stateful/rescalable pipeline built from
``dataset_utils`` (streaming docs -> logical shards -> corpus sampling -> packing -> shuffle
buffer -> tensor -> causal shift -> auto-checkpoint).
"""
from __future__ import annotations

import torch

from fms_fsdp_b200.utils import dataset_utils as D

_handler_map = {
    "arrow": D.ArrowHandler,
    "hf_parquet": D.ParquetHandler,
    "auto": D.AutoHandler,
}


def causal_lm(data_seq, prompt_len: int = 1):
    """(inputs, labels) = (x[:-1], x[1:]) with the first ``prompt_len`` labels masked to -100.
    Reference: ``fms_fsdp/utils/dataloader_utils.py:24-33``."""
    data_seq = data_seq.int() if isinstance(data_seq, torch.Tensor) else torch.IntTensor(data_seq)
    t = data_seq.clone()[1:]
    data_seq = data_seq[:-1]
    t[:prompt_len] = -100
    return data_seq, t


class _SteadyCounter(torch.utils.data.IterableDataset):
    """The reference's benchmarking stream (``dataloader_utils.py:36-57``, SURVEY Q8): sample k is the k-th window of
    ``seq_len`` consecutive integers modulo the vocabulary -- ``arange(k*seq, (k+1)*seq) % vocab`` -- so the stream
    sweeps the whole vocabulary; every rank yields the same samples and input == label (unshifted)."""

    def __init__(self, seq_len: int, vocab_size: int):
        self.seq_len, self.vocab_size = seq_len, vocab_size
        self.i = 0

    def __iter__(self):
        while True:
            t = (torch.arange(self.i, self.i + self.seq_len) % self.vocab_size).int()
            yield t, t
            self.i += self.seq_len


def get_dummy_loader(cfg, rank, world_size):
    """Reference: ``fms_fsdp/utils/dataloader_utils.py:36-57``."""
    return iter(torch.utils.data.DataLoader(_SteadyCounter(cfg.seq_length, cfg.vocab_size),
                                            batch_size=cfg.batch_size))


def parse_data_args(datas, weights):
    """'a,b,c' -> ['a','b','c'];  '1,2.5' -> [1.0, 2.5]  (reference :149-163)."""
    def split(x, cast):
        if isinstance(x, str):
            return [cast(v.strip()) for v in x.split(",") if v.strip() != ""]
        if isinstance(x, (list, tuple)):
            return [cast(v) for v in x]
        return [cast(x)]
    return split(datas, str), split(weights, float)


def get_data_loader(cfg, rank, world_size, postprocess=[causal_lm]):
    """Stateful, rescalable streaming loader. ``postprocess`` is applied after tensor conversion
    (the speculator passes [] to keep unshifted sequences).
    Reference: ``fms_fsdp/utils/dataloader_utils.py:60-146``."""
    datasets, weights = parse_data_args(cfg.datasets, cfg.weights)

    def _tok(x):
        return int(x) if x is not None and x != "" else None
    droplist = [int(x.strip()) for x in str(cfg.strip_tokens).split(",") if x.strip() != ""]
    droplist = droplist + [cfg.bos_token, cfg.eos_token, cfg.bol_token, cfg.eol_token]
    if cfg.file_type not in _handler_map:
        raise AssertionError(f"File type {cfg.file_type} is not recognized ({list(_handler_map.keys())})")
    if cfg.file_type == "hf_parquet":
        filehandler = D.ParquetHandler(cfg.tokenizer_path, cfg.col_name)
    elif cfg.file_type == "auto":
        filehandler = D.AutoHandler(cfg.tokenizer_path, cfg.col_name)
    else:
        filehandler = D.ArrowHandler(cfg.col_name)
    data = D.StreamingDocDataset(
        cfg.data_path, rank, world_size, filehandler, cfg.eos_token, bos_token=cfg.bos_token,
        strip_tokens=set(t for t in droplist if t is not None), min_length=3, seed=cfg.seed)
    data = D.ScalableShardDataset(data, cfg.eos_token, n_logical_shards=cfg.logical_shards)
    data = D.SamplingDataset(cfg.data_path, data, cfg.eos_token, datasets=datasets, weights=weights, verbose=(rank == 0))
    data = D.BufferDataset(data, cfg.seq_length if causal_lm not in postprocess else cfg.seq_length + 1,
                           bos_token=cfg.bol_token, eos_token=cfg.eol_token, pack_hard=True)
    data = D.PreloadBufferDataset(data, 10000)
    data = D.PreprocessDataset(data, torch.IntTensor)
    for p in postprocess:
        data = D.PreprocessDataset(data, p)
    # the loader counts optimizer steps (batch_size x grad_accum_steps sequences each), so its state is written at the
    # same steps as the model checkpoint
    data = D.CheckpointDataset(
        data, cfg.ckpt_load_path if cfg.resuming_dataset else cfg.ckpt_save_path,
        cfg.checkpoint_interval, cfg.batch_size * getattr(cfg, "grad_accum_steps", 1), cfg.ckpt_save_path)
    return torch.utils.data.DataLoader(data, num_workers=cfg.num_workers, batch_size=cfg.batch_size)

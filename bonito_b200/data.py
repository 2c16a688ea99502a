"""
Chunk datasets for `evaluate`, with the behaviour of the reference's bonito/data.py (host-only: numpy arrays behind
torch DataLoaders).

A data directory holds either
  * `chunks.npy` [N, L] (signal), `references.npy` [N, S] (labels 1..4, 0-padded) and `reference_lengths.npy` [N], with an
    optional `indices.npy` selecting and ordering the chunks and an optional `validation/` subdirectory of the same form;
    without `validation/` the last `valid_chunks` chunks of the training arrays are the validation set;
  * or a `dataset.py` whose `Loader(**settings)` provides `train_loader_kwargs(**settings)` and
    `valid_loader_kwargs(**settings)` (the settings include the model's standardisation and context bases).
"""

import importlib.util
import os
from dataclasses import dataclass
from pathlib import Path
from typing import Dict

import numpy as np
from torch.utils.data import DataLoader


@dataclass
class DataSettings:
    training_data: Path
    num_train_chunks: int
    num_valid_chunks: int
    output_dir: Path


@dataclass
class ComputeSettings:
    batch_size: int
    num_workers: int
    seed: int
    pin_memory: bool = True


@dataclass
class ModelSetup:
    n_pre_context_bases: int
    n_post_context_bases: int
    standardisation: Dict


class ChunkDataSet:
    """(chunk [1, L] float32, target [S] int64, length int64) per item."""

    def __init__(self, chunks, targets, lengths):
        self.chunks = np.expand_dims(chunks, axis=1)
        self.targets = targets
        self.lengths = lengths

    def __getitem__(self, i):
        return self.chunks[i].astype(np.float32), self.targets[i].astype(np.int64), self.lengths[i].astype(np.int64)

    def __len__(self):
        return len(self.lengths)


def load_numpy_datasets(limit=None, directory=None):
    """(chunks, targets, lengths) of one directory: the rows `indices.npy` lists (those below the chunk count, then the
    first `limit`), else the first `limit` rows (all with limit None or 0)."""
    arrays = [np.load(os.path.join(directory, name), mmap_mode="r")
              for name in ("chunks.npy", "references.npy", "reference_lengths.npy")]
    index_file = os.path.join(directory, "indices.npy")
    if os.path.exists(index_file):
        idx = np.load(index_file, mmap_mode="r")
        idx = idx[idx < arrays[2].shape[0]]
        if limit:
            idx = idx[:limit]
        return tuple(a[idx] for a in arrays)
    if limit:
        arrays = [a[:limit] for a in arrays]
    return tuple(np.array(a) for a in arrays)


def load_numpy(limit, directory, valid_chunks=None):
    """Loader kwargs (train shuffled, valid in order) of a chunks.npy directory."""
    train = load_numpy_datasets(limit=limit, directory=directory)
    valid_dir = os.path.join(directory, "validation")
    if os.path.exists(valid_dir):
        valid = load_numpy_datasets(limit=valid_chunks, directory=valid_dir)
    else:
        print("[validation set not found: splitting training set]")
        total = len(train[0])
        split = int(np.floor(total * 0.97)) if valid_chunks is None else max(0, total - valid_chunks)
        train, valid = tuple(a[:split] for a in train), tuple(a[split:] for a in train)
    # an empty training split (a directory that holds only the chunks to evaluate) is not shuffled: torch's RandomSampler
    # refuses an empty dataset
    train_set = ChunkDataSet(*train)
    return {"dataset": train_set, "shuffle": len(train_set) > 0}, {"dataset": ChunkDataSet(*valid), "shuffle": False}


def load_script(directory, name="dataset", suffix=".py", **kwargs):
    """Loader kwargs from `<directory>/dataset.py`'s Loader class."""
    path = (Path(directory) / name).with_suffix(suffix)
    spec = importlib.util.spec_from_file_location(name, path)
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    loader = module.Loader(**kwargs)
    return loader.train_loader_kwargs(**kwargs), loader.valid_loader_kwargs(**kwargs)


def load_data(data, model_setup, compute_settings):
    """(train DataLoader, valid DataLoader) for `data.training_data`; IOError when it cannot be loaded."""
    directory = Path(data.training_data)
    try:
        if (directory / "chunks.npy").exists():
            print(f"[loading data] - chunks from {directory}")
            train_kwargs, valid_kwargs = load_numpy(data.num_train_chunks, directory, valid_chunks=data.num_valid_chunks)
        elif (directory / "dataset.py").exists():
            print(f"[loading data] - dynamically from {directory}/dataset.py")
            train_kwargs, valid_kwargs = load_script(
                directory, chunks=data.num_train_chunks, valid_chunks=data.num_valid_chunks, log_dir=data.output_dir,
                n_pre_context_bases=model_setup.n_pre_context_bases, n_post_context_bases=model_setup.n_post_context_bases,
                standardisation=model_setup.standardisation, seed=compute_settings.seed,
                batch_size=compute_settings.batch_size, num_workers=compute_settings.num_workers)
        else:
            raise FileNotFoundError(f"No suitable training data found at: {directory}")
    except Exception as err:
        raise IOError(f"Failed to load input data from {directory}") from err
    defaults = {"batch_size": compute_settings.batch_size, "num_workers": compute_settings.num_workers,
                "pin_memory": compute_settings.pin_memory}
    # the script's loader kwargs override the defaults
    return DataLoader(**{**defaults, **train_kwargs}), DataLoader(**{**defaults, **valid_kwargs})

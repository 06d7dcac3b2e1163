"""A minimal import-level stand-in for `pytorch_lightning` (test infrastructure only).  It is NOT Lightning.

It lets the unmodified RecTools transformer models (rectools/models/nn/transformers/base.py, lightning.py) and the DSSM
module (rectools/models/nn/dssm.py) import, fit on small synthetic datasets and recommend, where the real package is not
installed.  It covers exactly these calls:

* `LightningModule`: a `torch.nn.Module` whose `save_hyperparameters` and `log` do nothing, with empty hooks
  (`on_train_start`, `on_train_end`, ...) and a `device` property;
* `Trainer(**kwargs)`: the keyword arguments are kept and ignored except `max_epochs`.  `fit(model, train_dataloader,
  val_dataloader=None)` (or Lightning's keywords `train_dataloaders=` / `val_dataloaders=`, as DSSM passes them) calls
  `model.configure_optimizers()` once and then, for each of `max_epochs` epochs, every batch of the loader (a dict of
  tensors, or a sequence of them) moved to the module's device: `zero_grad`, `training_step(batch, batch_idx)`,
  `backward`, `step`.  The
  hooks `on_train_start` / `on_train_end` run around that; validation loaders are not run.  `fit_loop.max_epochs`,
  `fit_loop.min_epochs` and `fit_loop.epoch_progress.current.ready` are kept as RecTools' `fit_partial` reads and sets them;
  `fit` continues from the ready epochs;
* `Callback`, `loggers.Logger`: empty placeholders;
* `seed_everything(seed)`: seeds Python, numpy and torch.

No precision, accelerator, distributed, checkpointing, logging or callback behaviour exists here."""
from __future__ import annotations

import random
import typing as tp
from types import SimpleNamespace

import numpy as np
import torch

from . import loggers  # noqa: F401

__version__ = "0.0.0+stub"


def seed_everything(seed: int = 0, workers: bool = False) -> int:  # pylint: disable=unused-argument
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    return seed


class Callback:
    """Placeholder: callbacks are accepted by nothing here."""


class LightningModule(torch.nn.Module):
    """`torch.nn.Module` with Lightning's bookkeeping calls as no-ops."""

    def save_hyperparameters(self, *args: tp.Any, **kwargs: tp.Any) -> None:
        pass

    def log(self, *args: tp.Any, **kwargs: tp.Any) -> None:
        pass

    @property
    def device(self) -> torch.device:
        p = next(self.parameters(), None)
        return p.device if p is not None else torch.device("cpu")

    def on_train_start(self) -> None:
        pass

    def on_train_end(self) -> None:
        pass

    def on_validation_start(self) -> None:
        pass

    def on_validation_end(self) -> None:
        pass


class Trainer:
    """`fit` runs plain optimisation epochs over the training loader (see the module docstring)."""

    def __init__(self, max_epochs: tp.Optional[int] = None, min_epochs: tp.Optional[int] = None, **kwargs: tp.Any) -> None:
        self.kwargs = kwargs
        self.fit_loop = SimpleNamespace(
            max_epochs=1 if max_epochs is None else int(max_epochs),
            min_epochs=min_epochs,
            epoch_progress=SimpleNamespace(current=SimpleNamespace(ready=0)),
        )

    @property
    def max_epochs(self) -> int:
        return self.fit_loop.max_epochs

    def fit(self, model: LightningModule, train_dataloader: tp.Any = None, val_dataloader: tp.Any = None, **kwargs: tp.Any) -> None:  # pylint: disable=unused-argument
        if train_dataloader is None:
            train_dataloader = kwargs.get("train_dataloaders")
        optimizer = model.configure_optimizers()
        if isinstance(optimizer, dict):
            optimizer = optimizer["optimizer"]
        elif isinstance(optimizer, (list, tuple)):
            optimizer = optimizer[0]
        device = model.device
        model.train()
        model.on_train_start()
        progress = self.fit_loop.epoch_progress.current
        while progress.ready < self.fit_loop.max_epochs:
            for batch_idx, batch in enumerate(train_dataloader or ()):
                if isinstance(batch, dict):
                    batch = {k: v.to(device) if hasattr(v, "to") else v for k, v in batch.items()}
                else:
                    batch = [v.to(device) if hasattr(v, "to") else v for v in batch]
                optimizer.zero_grad()
                loss = model.training_step(batch, batch_idx)
                loss.backward()
                optimizer.step()
            progress.ready += 1
        model.on_train_end()

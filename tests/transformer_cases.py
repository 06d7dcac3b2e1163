"""SASRec / BERT4Rec / HSTU built the way a user builds them, fitted on small synthetic datasets (shared by the CPU and GPU
tests of `install(transformers=True)`).  Needs the reference package and the `pytorch_lightning` stand-in on sys.path
(`oracle.stage_reference.add_to_path()`, `tests.lightning_stub.add_to_path()`).

The data preparators differ from the stock ones in one attribute only: `item_extra_tokens` is an object ndarray instead of
a tuple, because `IdMap.from_values` hands it to `pd.unique`, which takes no tuples from pandas 3 on.  The tokens and
their order are the stock ones."""
import numpy as np


from rectools.models.nn.transformers.bert4rec import BERT4RecDataPreparator  # noqa: E402
from rectools.models.nn.transformers.sasrec import SASRecDataPreparator  # noqa: E402


class ArraySASRecDataPreparator(SASRecDataPreparator):
    item_extra_tokens = np.array(SASRecDataPreparator.item_extra_tokens, dtype=object)


class ArrayBERT4RecDataPreparator(BERT4RecDataPreparator):
    item_extra_tokens = np.array(BERT4RecDataPreparator.item_extra_tokens, dtype=object)


MODELS = ("sasrec", "bert4rec", "hstu")


def build_model(name, n_factors=16, epochs=2, device="cpu", seed=0):
    """An unfitted model: SASRec (DOT), BERT4Rec (DOT, PAD + MASK tokens) or HSTU (COSINE)."""
    import torch
    from rectools.models import BERT4RecModel, HSTUModel, SASRecModel

    torch.manual_seed(seed)
    np.random.seed(seed)
    sas_prep, bert_prep = ArraySASRecDataPreparator, ArrayBERT4RecDataPreparator
    common = dict(n_factors=n_factors, n_blocks=1, n_heads=1, session_max_len=8, epochs=epochs, batch_size=64,
                  recommend_torch_device=device, deterministic=True)
    if name == "sasrec":
        return SASRecModel(data_preparator_type=sas_prep, **common)
    if name == "bert4rec":
        return BERT4RecModel(data_preparator_type=bert_prep, **common)
    if name == "hstu":
        # (relative time attention needs a recommendation context: off, so that recommend() takes the usual arguments)
        return HSTUModel(data_preparator_type=sas_prep, similarity_module_kwargs={"distance": "cosine"}, relative_time_attention=False,
                         **common)
    raise ValueError(name)


def dataset(n_users=80, n_items=150, per_user=12, seed=1):
    """`tests.ref_models.synthetic_dataset` plus one user (external id 1) who has viewed every item."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset

    from tests.ref_models import synthetic_dataset

    base = synthetic_dataset(n_users, n_items, per_user, seed=seed)
    df = base.interactions.to_external(base.user_id_map, base.item_id_map)
    every = pd.DataFrame({Columns.User: 1, Columns.Item: base.item_id_map.external_ids, Columns.Weight: 1.0,
                          Columns.Datetime: pd.Timestamp("2024-01-02")})
    return Dataset.construct(pd.concat([df, every], ignore_index=True))

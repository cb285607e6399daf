"""financial_market_data_analysis_b200 - H100-native (sm_90a) implementation of the one hot path of
radoslawkrolikowski/financial-market-data-analysis: the bidirectional-GRU classifier
(biGRU_model.py) and the windowed collation that feeds it (sql_pytorch_dataloader.py).

The two sub-modules keep the reference's module names so that putting this directory on
sys.path makes ``from biGRU_model import BiGRU`` / ``from sql_pytorch_dataloader import ...``
(predict.py:16, the training notebook) resolve to the CUDA implementation.
"""
from . import _lib
from .biGRU_model import BiGRU
from .sql_pytorch_dataloader import (MySQLBatchLoader, MySQLChunkLoader, TrainValTestSplit,
                                     window_indices)

__all__ = ["BiGRU", "MySQLBatchLoader", "MySQLChunkLoader", "TrainValTestSplit", "window_indices", "_lib"]

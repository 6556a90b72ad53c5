"""models_b200 — H100-native (sm_90a) implementation of the Merlin Models hot path:
embedding lookup -> MLP tower -> interaction / scoring, behind the reference's constructors.

    import models_b200 as mm
    model = mm.DLRMModel(schema, embedding_dim=64, bottom_block=mm.MLPBlock([128, 64]),
                         top_block=mm.MLPBlock([128, 64, 32]))
    logits = model(features)          # dict of CUDA tensors -> (B, 1) fp32

Importing the package does not need a GPU (constructors, schema handling); calling a block
does — there is no CPU fallback (see oracle/ for the CPU restatement used by the tests).
"""
from .schema import ColumnSchema, Schema, Tags  # noqa: F401
from .core import Block, Prediction, PredictionOutput, SequentialBlock, set_seed, to_device  # noqa: F401
from .inputs import (ContinuousFeatures, EmbeddingOptions, Embeddings, EmbeddingTable, InputBlock,  # noqa: F401
                     InputBlockV2, infer_embedding_dim)
from .blocks import (CrossBlock, DLRMBlock, DotProductInteraction, MLPBlock, dense_engine,  # noqa: F401
                     set_dense_engine)
from .blocks import BatchNormalization, CategoryEncoding, FMBlock, FMPairwiseInteraction, HashedCross, HashedCrossAll  # noqa: F401
from .experts import CGCBlock, MMOEBlock, PLEBlock  # noqa: F401
from .retrieval import (CategoricalOutput, ContrastiveOutput, Encoder, InBatchSampler, InBatchSamplerV2,  # noqa: F401
                        ItemRetrievalScorer, ItemRetrievalTask, L2Norm, PopularityBasedSamplerV2,
                        QueryItemIdsEmbeddingsBlock, TwoTowerBlock, log_uniform_sampling_probs)
from .models import (BinaryClassificationTask, BinaryOutput, CatalogModel, DCNModel, DeepFMModel, DLRMModel, Model, OutputBlock,  # noqa: F401
                     ParallelOutputs, RegressionOutput, WideAndDeepModel,
                     MatrixFactorizationModel, RetrievalModel, RetrievalModelV2, TwoTowerModel, TwoTowerModelV2)
from .topk import (AvgPrecisionAt, BruteForce, MRRAt, NDCGAt, PrecisionAt, RecallAt, TopKEncoder,  # noqa: F401
                   TopKIndexBlock, TopKPrediction, encode_candidates, unique_rows_by_features)
from .loader import Loader, sample_batch  # noqa: F401
from .pretrained import EmbeddingOperator, PretrainedEmbeddings, TensorInitializer  # noqa: F401
from .graph import CompiledForward, HostBatch, PipelinedForward  # noqa: F401
from .sharded import ShardedEmbeddings, shard_model  # noqa: F401
from .train import SGD, Adagrad, Adam, DLRMTrainer, LazyAdam  # noqa: F401
from .optimizer import MultiOptimizer, OptimizerBlocks, split_embeddings_on_size  # noqa: F401
from . import benchmark, datasets, io, losses, metrics, ops, schedules, train  # noqa: F401
from .io import load_merlin_metadata, save_merlin_metadata  # noqa: F401

__version__ = "0.1.0"

"""merlin/models/tf/models/benchmark.py: the neural collaborative filtering model (NCFModel), exported as
`mm.benchmark.NCFModel` like the reference's."""
from __future__ import annotations

from typing import Optional

from .blocks import MLP
from .models import BinaryOutput, NCFBody, OutputBlock, ParallelOutputs, RankingModel, parse_prediction_blocks
from .retrieval import QueryItemIdsEmbeddingsBlock
from .schema import Schema


def NCFModel(schema: Schema, embedding_dim: int, mlp_block: MLP, prediction_tasks=None, embeddings_l2_reg: float = 0.0,
             **kwargs) -> RankingModel:
    """models/benchmark.py:32-100 (He et al., "Neural Collaborative Filtering", arXiv:1708.05031): a RankingModel over
    NCFBody = concat([mf, mlp]) with
      mf   the GMF branch, user-id embedding * item-id embedding (MatrixFactorizationBlock with ElementWiseMultiply);
      mlp  mlp_block over [item-id embedding | user-id embedding] of a second, separate pair of tables;
    then the prediction blocks of `prediction_tasks` (default: OutputBlock(schema), one output per target column).  Every table is
    `embedding_dim` wide.  **kwargs (query_id_tag, item_id_tag, embeddings_initializers) reach the mf branch only, as in
    the reference: the mlp branch always embeds the USER_ID / ITEM_ID columns with the default initializer.
    embeddings_l2_reg adds embeddings_l2_reg * sum ||e||^2 over the batch's looked-up rows of all four tables to the loss."""
    if kwargs.get("post") is not None:
        raise NotImplementedError("NCFModel: a post block on the mf branch is not implemented")
    kwargs.pop("post", None)
    mlp_ids = QueryItemIdsEmbeddingsBlock(schema, dim=embedding_dim, embeddings_l2_reg=embeddings_l2_reg)
    mf = QueryItemIdsEmbeddingsBlock(schema, dim=embedding_dim, embeddings_l2_reg=embeddings_l2_reg, **kwargs)
    # the reference's parse_prediction_blocks(schema, None) is OutputBlock(schema): one output per target column
    prediction = OutputBlock(schema) if prediction_tasks is None else parse_prediction_blocks(schema, prediction_tasks)
    for o in (prediction.outputs if isinstance(prediction, ParallelOutputs) else [prediction]):
        if not isinstance(o, BinaryOutput):
            raise NotImplementedError(f"NCFModel: output {o.name!r} is not a BinaryOutput / RegressionOutput (the head kernel "
                                      "runs 1..8 of those)")
    return RankingModel(NCFBody(mf, mlp_ids, mlp_block, embeddings_l2_reg), prediction, schema)

"""Row-sharded embedding tables across the GPUs of one box (BASELINE config 4, SURVEY §8(e)).

Partitioning: row r of every sharded table lives on rank `r % world` at local row `r // world`
(balanced under skew).  Tables with fewer than `replicate_below_rows` rows (default 65 536 = 16 MB at
D = 64) are kept whole on every rank (SURVEY §8(e): "replicate tables with <= 64 k rows and shard only
the big ones"): a table of a handful of rows has nothing to shard, and sharding it anyway makes every
sample of every GPU read the same few cache lines of one owner over NVLink (the 8 tables under 1 000 rows
of the Criteo-TB shape are such tables).  `replicate_below_rows=0` shards everything.  Dense / MLP / interaction
weights are replicated; the batch is sharded data-parallel.

Forward (one process per GPU): all shards live in ONE symmetric-memory arena per rank
(`torch.distributed._symmetric_memory`: every rank maps every other rank's arena over NVLink, same
offsets everywhere).  The lookup is then part of the interaction kernel itself
(`mm_dlrm_lookup_interact`, csrc/interaction_v2.cu): for each (sample, table) the owning lane derives
owner = id % world, local row = id // world, and the cp.async that stages the row into shared memory
reads it from that rank's shard — local HBM or a peer's HBM over NVLink.  There is no index exchange,
no send/receive buffer, no collective and no barrier on the data path (tables are read-only in the
forward pass), so the sharded step is the same 4 launches as the replicated one and captures into a
CUDA graph like it.

The reference's counterpart is SOK's distributed variable + `sok.lookup_sparse`
(merlin/models/tf/distributed/embedding.py:75-84,144-148: all-to-all of keys, local lookup, all-to-all
of vectors).  The round-1 protocol — all-gather of the ids, owner-computes push into the
destination rank's (B_local, F, D) stack (`mm_shard_gather_push`), barrier — is kept as
`lookup_stack` (it is what a NCCL-style exchange looks like on the same shards and serves as the
baseline the fused kernel is measured against).  Host logic here (ownership maths, index all-gather,
stack layout) is backend-agnostic and covered by world-size-2 gloo tests on CPU; the device step
needs CUDA + peer access.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import _cabi, ops
from .core import create_variable
from .inputs import EmbeddingsBlock


# ---- ownership maths (pure, also used by the tests) -------------------------------------------------
def owner_of(idx: torch.Tensor, world: int) -> torch.Tensor:
    """Rank that owns global row `idx` (Python modulo semantics: negative ids map into 0..world-1)."""
    return torch.remainder(idx, world)


def local_row(idx: torch.Tensor, world: int) -> torch.Tensor:
    return torch.div(idx, world, rounding_mode="floor")


def local_row_count(rows: int, rank: int, world: int) -> int:
    """Number of global rows r in [0, rows) with r % world == rank."""
    return (rows - rank + world - 1) // world if rows > rank else 0


def shard_of(full: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """The rows of a full table owned by `rank` (global rows rank, rank+world, ...)."""
    return full[rank::world].contiguous()


class ShardedEmbeddings:
    """Local shards of every table of an EmbeddingsBlock inside one symmetric-memory arena, the peer
    pointers of every other rank's arena, and the fused lookup + interaction launch."""

    def __init__(self, embeddings: EmbeddingsBlock, group=None, device=None, replicate_below_rows: int = 65536):
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.embeddings = embeddings
        self.device = device
        self.replicate_below_rows = int(replicate_below_rows)
        self.feature_names: List[str] = embeddings.feature_names
        dims = set(embeddings.output_dims().values())
        if len(dims) != 1:
            raise ValueError("sharded lookup needs one embedding dimension for all tables")
        self.D = dims.pop()
        self.shards: Dict[str, torch.Tensor] = {}     # table name -> local shard (or the whole table if replicated)
        self.peer_ptrs: Dict[str, Optional[List[int]]] = {}  # table name -> device pointers of every rank's shard (None: replicated)
        self.global_rows: Dict[str, int] = {n: t.input_dim for n, t in embeddings.tables.items()}
        self.arena = None
        self._arena_hdl = None
        self._offsets: Dict[str, int] = {}
        self.mirrors: Dict[str, torch.Tensor] = {}   # table name -> shard / table as bf16 split rows (ops.split_rows)
        self.mirror_peer_ptrs: Dict[str, Optional[List[int]]] = {}
        self.mirror_arena = None
        self._mirror_hdl = None
        self._symm = None
        self._symm_key = None

    def is_sharded(self, table_name: str) -> bool:
        return self.world > 1 and self.global_rows[table_name] >= self.replicate_below_rows

    # ---- shard construction -------------------------------------------------------------------------
    def _allocate(self, device):
        """One arena for all sharded tables (same offsets on every rank) + plain tensors for replicated ones."""
        if self.shards:
            return
        self.device = device
        D = self.D
        off, offsets = 0, {}
        for name, table in self.embeddings.tables.items():
            if self.is_sharded(name):
                offsets[name] = off
                lrows_max = (table.input_dim + self.world - 1) // self.world  # same on every rank
                off += ((max(lrows_max, 1) * D + 63) // 64) * 64  # 256-B aligned shards
        self._offsets, self._arena_floats = offsets, off
        arena_ptrs = None
        if off and device.type == "cuda":
            import torch.distributed._symmetric_memory as symm_mem

            self.arena = symm_mem.empty((off,), dtype=torch.float32, device=device)
            self._arena_hdl = symm_mem.rendezvous(self.arena, group=self.group)
            arena_ptrs = [int(p) for p in self._arena_hdl.buffer_ptrs]
        elif off:
            self.arena = torch.empty((off,), dtype=torch.float32, device=device)  # CPU (gloo tests): no peer mapping
        for name, table in self.embeddings.tables.items():
            if name in offsets:
                lrows = local_row_count(table.input_dim, self.rank, self.world)
                o = offsets[name]
                self.shards[name] = self.arena[o: o + max(lrows, 1) * D].view(max(lrows, 1), D)
                self.peer_ptrs[name] = None if arena_ptrs is None else [p + 4 * o for p in arena_ptrs]
            else:
                self.shards[name] = torch.empty((table.input_dim, D), dtype=torch.float32, device=device)
                self.peer_ptrs[name] = None

    def _maybe_mirror(self):
        from .blocks import table_mirror

        if table_mirror() and self.device is not None and self.device.type == "cuda" and self.D == 64:
            self.build_mirrors()

    def _publish(self):
        """Shards are written once; every rank must see every other rank's rows before the first lookup."""
        if self.device is not None and self.device.type == "cuda":
            torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=self.group)

    def build(self, device) -> "ShardedEmbeddings":
        """Create the local shard of every table directly (never materialising a full sharded table)."""
        if self.shards:
            return self
        self._allocate(device)
        for name, table in self.embeddings.tables.items():
            w = self.shards[name]
            init = table.embeddings_initializer
            shd = self.is_sharded(name)
            lrows = local_row_count(table.input_dim, self.rank, self.world) if shd else table.input_dim
            if isinstance(init, dict) and "hash_seed" in init:
                _cabi.check(_cabi.load().mm_init_uniform_hash_rows(
                    w.data_ptr(), lrows, table.dim, init["hash_seed"] & (2**64 - 1), init.get("lo", -0.05),
                    init.get("hi", 0.05), self.rank if shd else 0, self.world if shd else 1,
                    torch.cuda.current_stream().cuda_stream), "mm_init_uniform_hash_rows")
            elif isinstance(init, (torch.Tensor,)) or hasattr(init, "shape"):
                full = torch.as_tensor(init, dtype=torch.float32)
                w[:lrows].copy_(shard_of(full, self.rank, self.world) if shd else full)
            else:
                # seeded generators are rank-independent: build the full table, keep this rank's rows
                full = create_variable((table.input_dim, table.dim), init, device, f"{table.table_name}/embeddings")
                w[:lrows].copy_(shard_of(full, self.rank, self.world) if shd else full)
                del full
        self._publish()
        self._maybe_mirror()
        return self

    def load_full_tables(self, full: Dict[str, torch.Tensor], device) -> "ShardedEmbeddings":
        """Shard explicitly given full tables (tests, checkpoints)."""
        self._allocate(device)
        for name in self.embeddings.tables:
            src = torch.as_tensor(full[name], dtype=torch.float32)
            if self.is_sharded(name):
                mine = shard_of(src, self.rank, self.world)
                self.shards[name][: mine.shape[0]].copy_(mine)
                self.shards[name] = self.shards[name][: max(mine.shape[0], 1)]
            else:
                self.shards[name].copy_(src)
        self._publish()
        self._maybe_mirror()
        return self

    def build_mirrors(self) -> None:
        """Operand-format copies of every shard (a second symmetric arena, same offsets: peers read the MIRROR rows over
        NVLink) and of every replicated table.  Collective over the group (rendezvous + barrier); idempotent."""
        if self.mirrors or not self.shards:
            return
        dev = self.device
        arena_ptrs = None
        if self._arena_floats and dev.type == "cuda":
            import torch.distributed._symmetric_memory as symm_mem

            self.mirror_arena = symm_mem.empty((2 * self._arena_floats,), dtype=torch.bfloat16, device=dev)
            self._mirror_hdl = symm_mem.rendezvous(self.mirror_arena, group=self.group)
            arena_ptrs = [int(p) for p in self._mirror_hdl.buffer_ptrs]
        for name, shard in self.shards.items():
            if name in self._offsets and self.mirror_arena is not None:
                o = self._offsets[name]
                view = self.mirror_arena[2 * o: 2 * o + 2 * shard.numel()].view(shard.shape[0], 2 * shard.shape[1])
                ops.split_rows(shard, out=view)
                self.mirrors[name] = view
                self.mirror_peer_ptrs[name] = [p + 4 * o for p in arena_ptrs]
            else:
                self.mirrors[name] = ops.split_rows(shard.contiguous())
                self.mirror_peer_ptrs[name] = None
        self._publish()

    # ---- the product path: lookup fused into the interaction kernel ----------------------------------
    def lookup_interact(self, local_inputs: Dict[str, torch.Tensor], slots: Dict[str, int], bottom: Optional[torch.Tensor],
                        out: torch.Tensor, oob: Optional[torch.Tensor] = None, operand_rows: bool = False) -> torch.Tensor:
        """out = [bottom | pairwise dots] of this rank's samples; rows owned by other ranks are read over
        NVLink inside the kernel (mm_dlrm_lookup_interact).  operand_rows: `bottom` is in operand format and the
        operand-format mirrors of the shards are read (build_mirrors must have run — ShardedEmbeddings.build does it
        when the table mirrors are enabled)."""
        if not self.shards:
            raise RuntimeError("ShardedEmbeddings.build(device) must be called first")
        from .core import get_feature

        names = [self.embeddings.feature_to_table[f].table_name for f in self.feature_names]
        idx = [ops.fused_ids(get_feature(local_inputs, f)) for f in self.feature_names]
        if operand_rows and not self.mirrors:
            raise RuntimeError("operand-format rows requested but build_mirrors() has not run")
        tabs = self.mirrors if operand_rows else self.shards
        pp = self.mirror_peer_ptrs if operand_rows else self.peer_ptrs
        return ops.dlrm_lookup_interact(
            [tabs[n] for n in names], idx, [slots[f] for f in self.feature_names], [self.global_rows[n] for n in names],
            self.D, bottom, slots.get("bottom_block", -1), out, oob,
            peers=[pp[n] if self.is_sharded(n) else None for n in names], rank=self.rank, world=self.world,
            operand_rows=operand_rows)

    # ---- step 1: replicate the indices ----------------------------------------------------------------
    def gather_indices(self, local_inputs: Dict[str, torch.Tensor]) -> torch.Tensor:
        """(T, B_local) local -> (T, world*B_local) global, rank-major sample order."""
        idx = torch.stack([ops.as_index(local_inputs[f]).reshape(-1) for f in self.feature_names], dim=0).contiguous()
        if len({ops.as_index(local_inputs[f]).dtype for f in self.feature_names}) > 1:
            idx = idx.to(torch.int64)
        T, Bl = idx.shape
        out = torch.empty((self.world, T, Bl), dtype=idx.dtype, device=idx.device)
        dist.all_gather(list(out.unbind(0)), idx, group=self.group)  # works on NCCL and gloo alike
        return out.permute(1, 0, 2).reshape(T, self.world * Bl).contiguous()

    # ---- step 2 + 3: owner-computes push over peer memory, then barrier ------------------------------
    def _stack_buffer(self, B_local: int, width: int):
        """Symmetric (peer-mapped) fp32 buffer (B_local, width) + every rank's pointer to it."""
        key = (B_local, width)
        if self._symm_key != key:
            import torch.distributed._symmetric_memory as symm_mem

            buf = symm_mem.empty((B_local, width), dtype=torch.float32, device=self.device)
            hdl = symm_mem.rendezvous(buf, group=self.group)
            self._symm = (buf, hdl, [int(p) for p in hdl.buffer_ptrs])
            self._symm_key = key
        return self._symm

    def lookup_stack(self, local_inputs: Dict[str, torch.Tensor], slots: Dict[str, int], n_slots: int,
                     oob: Optional[torch.Tensor] = None) -> torch.Tensor:
        """(B_local, n_slots*D) stack with feature f at slot slots[f] (other slots untouched)."""
        if not self.shards:
            raise RuntimeError("ShardedEmbeddings.build(device) must be called first")
        if any(not self.is_sharded(n) for n in self.shards) and self.world > 1:
            raise NotImplementedError("lookup_stack (push protocol) needs every table sharded (replicate_below_rows=0)")
        g_idx = self.gather_indices(local_inputs)
        T, Bg = g_idx.shape
        Bl = Bg // self.world
        D = self.D
        buf, hdl, ptrs = self._stack_buffer(Bl, n_slots * D)
        arr = (_cabi.GatherTable * T)()
        for t, f in enumerate(self.feature_names):
            table = self.embeddings.feature_to_table[f]
            shard = self.shards[table.table_name]
            arr[t].weights = shard.data_ptr()
            arr[t].indices = g_idx[t].data_ptr()
            arr[t].rows = self.global_rows[table.table_name]
            arr[t].dim = D
            arr[t].out_col = slots[f] * D
        dst = (C.c_void_p * self.world)(*ptrs)
        hdl.barrier(channel=0)  # every rank is done reading the previous batch's stack
        _cabi.check(
            _cabi.load().mm_shard_gather_push(arr, T, ops._idx_dtype(g_idx, "indices"), Bg, Bl, D, self.rank, self.world,
                                              dst, n_slots * D, None if oob is None else oob.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream),
            "mm_shard_gather_push")
        hdl.barrier(channel=1)  # all pushes have landed
        return buf


def lookup_stack_nccl(se: "ShardedEmbeddings", local_inputs: Dict[str, torch.Tensor], slots: Dict[str, int], n_slots: int) -> torch.Tensor:
    """BASELINE, not a product path: the row-sharded lookup the way the north star words it and the way a PyTorch/NCCL
    program (or SOK's lookup_sparse, distributed/embedding.py:75-84,144-148) does it — all-gather of the ids, a local gather
    of the owned rows packed by destination rank, ONE variable-size NCCL all-to-all of the vectors (split sizes exchanged
    first and read back on the host, as `all_to_all_single` needs them), then a scatter into the (B_local, n_slots*D)
    stack.  Written with torch ops + torch.distributed on purpose: it is what the fused peer-memory kernel is measured
    against (bench.py `sharded.nccl_all_to_all_ms`), and tests/dist_sharded_check.py checks that both give the same rows.
    Replicated tables are looked up locally."""
    W, rank, D = se.world, se.rank, se.D
    names = [(f, se.embeddings.feature_to_table[f].table_name) for f in se.feature_names]
    sharded = [(f, n) for f, n in names if se.is_sharded(n)]
    dev = next(iter(local_inputs.values())).device
    Bl = ops.as_index(local_inputs[se.feature_names[0]]).reshape(-1).shape[0]
    stack = torch.zeros((Bl, n_slots * D), dtype=torch.float32, device=dev)
    for f, n in names:
        if not se.is_sharded(n):
            stack.view(Bl, n_slots, D)[:, slots[f]] = se.shards[n][ops.as_index(local_inputs[f]).reshape(-1).long()]
    if not sharded:
        return stack
    ids = torch.stack([ops.as_index(local_inputs[f]).reshape(-1).long() for f, _ in sharded], dim=1).contiguous()  # (Bl, Ts)
    Ts = ids.shape[1]
    gids = torch.empty((W, Bl, Ts), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(gids.view(-1), ids.view(-1), group=se.group)
    mine = (gids % W) == rank                                   # entries of every rank's batch whose row I own
    send_counts = mine.view(W, -1).sum(dim=1)
    recv_counts = torch.empty_like(send_counts)
    dist.all_to_all_single(recv_counts, send_counts, group=se.group)
    in_splits, out_splits = send_counts.tolist(), recv_counts.tolist()   # host sync: all_to_all_single needs python ints
    w_idx, b_idx, t_idx = mine.nonzero(as_tuple=True)                    # sorted by destination rank, then (sample, table)
    lrow = gids[w_idx, b_idx, t_idx] // W
    send = torch.empty((int(w_idx.numel()), D), dtype=torch.float32, device=dev)
    for j, (_, n) in enumerate(sharded):
        sel = t_idx == j
        send[sel] = se.shards[n][lrow[sel]]
    recv = torch.empty((int(sum(out_splits)), D), dtype=torch.float32, device=dev)
    dist.all_to_all_single(recv, send, output_split_sizes=out_splits, input_split_sizes=in_splits, group=se.group)
    owner = ids % W                                                       # who sent me which of my (sample, table) entries
    col = torch.tensor([slots[f] for f, _ in sharded], device=dev)
    view = stack.view(Bl, n_slots, D)
    off = 0
    for r in range(W):
        b_r, t_r = (owner == r).nonzero(as_tuple=True)
        view[b_r, col[t_r]] = recv[off: off + b_r.numel()]
        off += b_r.numel()
    return stack


def shard_model(model, group=None, replicate_below_rows: int = 65536):
    """Row-shard the embedding tables of a DLRM model over `group` (call before the first forward;
    every rank then holds 1/world of each sharded table; tables with fewer than `replicate_below_rows`
    rows stay whole on every rank).  Returns the model."""
    from .blocks import DLRM

    body = getattr(model, "body", model)
    if not isinstance(body, DLRM):
        raise NotImplementedError("shard_model supports DLRM bodies")
    if any(t.table is not None for t in body.embeddings.tables.values()):
        raise RuntimeError("shard_model must be called before the tables are built")
    body.sharded = ShardedEmbeddings(body.embeddings, group, replicate_below_rows=replicate_below_rows)
    return model

"""One process per GPU: the dynamic resident state sharded by top key nibble (SURVEY.md §8e, DESIGN.md §8b).

Rank r of `world` owns the accounts whose hashed address starts with a nibble in [16r/world, 16(r+1)/world) together with
their storage tries.  A block's HashedPostState is filtered to the rank's buckets and committed to the local
`b200_dstate` shard; the ranks then all-gather their 16 frontier entries (16 x 68 bytes, torch.distributed: NCCL on
GPUs, gloo in the CPU tests) and every rank finishes the state root with b200_root_from_frontier.  No other data moves
between ranks: this is the collective-free partitioning of the reference's ParallelStateRoot fan-out
(crates/trie/parallel/src/root.rs:101-127) carried over to the live path."""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from .engine import Engine
from .hashed_state import HashedPostState, HashedPostStateSorted
from .trie import DynamicStateRoot, StateRootError, TrieUpdates, apply_layout


def owner_of(key: bytes, world: int) -> int:
    return (key[0] >> 4) * world // 16


class ShardedDynamicStateRoot:
    def __init__(self, engine: Engine, state: HashedPostState, rank: int, world: int, group=None, comm=None):
        """state: the full initial hashed state (every rank may pass the same object; only its buckets are kept) or
        already just this rank's part.  comm: a reth_b200.Comm — the frontier exchange then runs inside the library
        (b200_dstate_root_sharded, NCCL) instead of through torch.distributed."""
        if 16 % world and world > 16:
            raise ValueError("at most 16 ranks (one top-nibble bucket each)")
        self.engine, self.rank, self.world, self.group, self.comm = engine, rank, world, group, comm
        mine = HashedPostState({k: a for k, a in state.accounts.items() if owner_of(k, world) == rank},
                               {k: s for k, s in state.storages.items() if owner_of(k, world) == rank})
        self.local = DynamicStateRoot(engine, mine.into_sorted(), sharded=True)
        self._root = self._gather_root()

    def root(self) -> bytes:
        return self._root

    def _all_gather(self, fr: np.ndarray) -> np.ndarray:
        """fr: this rank's frontier rows (..., 16, 68) uint8 -> (world, ..., 16, 68), every rank's (torch.distributed)."""
        if self.world == 1:
            return fr[None]
        import torch
        import torch.distributed as dist
        dev = "cuda" if dist.get_backend(self.group) == "nccl" else "cpu"
        mine = torch.from_numpy(np.ascontiguousarray(fr).reshape(-1)).to(dev)
        gathered = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(gathered, mine, group=self.group)
        return torch.stack(gathered).cpu().numpy().reshape((self.world,) + fr.shape)

    def _merged_root(self, allf: np.ndarray) -> bytes:
        """allf: (world, 16, 68), every rank's entries -> the state root from the owner's entry of every bucket."""
        pick = np.arange(16) * self.world // 16                       # owner of every bucket (same map as bench.py)
        return self.engine.root_from_frontier(np.ascontiguousarray(allf[pick, np.arange(16)]))

    def _gather_root(self) -> bytes:
        if self.comm is not None:
            return self.comm.dstate_root_sharded(self.local.ds)
        fr = self.local.ds.frontier()                                  # (16, 68) uint8, empty outside this rank's buckets
        if self.world == 1:
            return self.engine.root_from_frontier(fr)
        return self._merged_root(self._all_gather(fr))

    def _part(self, post: HashedPostState) -> HashedPostState:
        return HashedPostState({k: a for k, a in post.accounts.items() if owner_of(k, self.world) == self.rank},
                               {k: s for k, s in post.storages.items() if owner_of(k, self.world) == self.rank})

    def commit(self, post: HashedPostState) -> Tuple[bytes, TrieUpdates]:
        """-> (state root, this rank's part of the block's TrieUpdates)."""
        _, updates = self.local.commit(self._part(post))
        self._root = self._gather_root()
        return self._root, updates

    def overlay_roots(self, posts) -> List[bytes]:
        """The state root `commit` of each post alone would return, with every shard left as it is: payload validation and
        payload building over a sharded state, before `commit` keeps one block (DynamicStateRoot.overlay_roots on one
        GPU).  The posts are siblings on the current state, not a chain.  Collective: every rank calls it with the same
        posts.  Each rank computes its frontier entries after every post (b200_dstate_overlay_frontiers), one all-gather of
        n x 16 x 68 bytes over torch.distributed exchanges them, and every rank finishes each root with
        b200_root_from_frontier.  At world > 1 a torch.distributed process group must be initialised, also when the
        object was made with `comm`: this exchange does not run through the library's NCCL communicator."""
        if not posts:
            return []
        blocks = [apply_layout(self._part(post), destroyed_slots=False)[1] for post in posts]
        try:
            fr = self.local.ds.overlay_frontiers(blocks)               # (n, 16, 68)
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        allf = self._all_gather(fr)                                    # (world, n, 16, 68)
        return [self._merged_root(allf[:, b]) for b in range(len(posts))]

    def overlay_root(self, post: HashedPostState) -> bytes:
        """overlay_roots for one post: the state root `commit(post)` would return, without changing any shard."""
        return self.overlay_roots([post])[0]

    def _gather_root_branch(self, extra: np.ndarray):
        """One all-gather of every rank's 16 x 68 frontier bytes, its 4 root-mask bytes and `extra` (uint8) -> (merged (16, 68):
        the owner's entry of every bucket, hash mask, tree mask, (world, len(extra)) every rank's extra bytes)."""
        ds = self.local.ds
        try:
            hm, tm = ds.frontier_masks()
            mine = np.concatenate([ds.frontier().reshape(-1), np.array([hm, tm], "<u2").view(np.uint8), extra])
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        allf = self._all_gather(mine)                                  # (world, 16 x 68 + 4 + len(extra))
        masks = allf[:, 16 * 68:16 * 68 + 4].copy().view("<u2")        # (world, 2)
        hash_mask, tree_mask = (int(np.bitwise_or.reduce(masks[:, i])) for i in range(2))
        frs = allf[:, :16 * 68].reshape(self.world, 16, 68)
        merged = np.ascontiguousarray(frs[np.arange(16) * self.world // 16, np.arange(16)])   # owner's entry of every bucket
        return merged, hash_mask, tree_mask, allf[:, 16 * 68 + 4:]

    def _answering_rank(self, merged: np.ndarray):
        """key -> the rank that answers it: the owner of its top nibble, or in the one-bucket case of that bucket"""
        nonempty = [k for k in range(16) if merged[k, 34]]             # as_root_len
        def owner(key: bytes) -> int:
            k = key[0] >> 4
            if k not in nonempty and len(nonempty) == 1:
                k = nonempty[0]
            return k * self.world // 16
        return owner

    def multiproof(self, targets: dict) -> dict:
        """Proof::multiproof(MultiProofTargets) of the whole state: eth_getProof and the proof workers of the state-root task
        over a sharded state.  targets: {hashed address: iterable of hashed slots}.  -> on every rank, the dict
        DynamicState.multiproof gives on one GPU.  Collective: every rank calls it with the same targets.  One all-gather
        of every rank's 16 x 68 frontier bytes and its 4 root-mask bytes gives the root branch; each target goes to the
        owner of its top nibble (in the one-bucket case, to that bucket's owner), each rank proves its share
        (b200_dstate_sharded_multiproof), and one all_gather_object of the partial dicts is merged.  At world > 1 a
        torch.distributed process group must be initialised, also when the object was made with `comm`."""
        ds = self.local.ds
        merged, hash_mask, tree_mask, _ = self._gather_root_branch(np.zeros(0, np.uint8))
        owner = self._answering_rank(merged)
        share = {a: s for a, s in targets.items() if owner(bytes(a)) == self.rank}
        try:
            part = ds.sharded_multiproof(merged, hash_mask, tree_mask, share)
        except ValueError:
            raise
        except Exception as e:  # noqa: BLE001
            raise StateRootError(str(e)) from e
        if self.world == 1:
            return part
        import torch.distributed as dist
        parts = [None] * self.world
        dist.all_gather_object(parts, part, group=self.group)
        out = {"account_subtree": {}, "branch_node_masks": {}, "storages": {}}
        for p in parts:
            for name in out:
                out[name].update(p[name])
        return out

    def witness(self, post: HashedPostState, mode: str = "legacy", always_include_root_node: bool = False) -> Dict[bytes, bytes]:
        """TrieWitness::compute(post) of the whole state (debug_executionWitness, the invalid-block witness hook, stateless
        clients) over a sharded state.  -> on every rank, the dict DynamicStateRoot.witness gives on one GPU; no shard
        changes.  Raises StateRootError for a storage entry without an account entry.  Collective: every rank calls it with
        the same post.  Each rank computes the kept mask of the block's entries in its own buckets
        (b200_dstate_witness_root_kept); one all-gather carries it with the 16 x 68 frontier bytes, the 4 root-mask bytes and
        a status byte; each entry then goes to the rank that answers it (as in `multiproof`; with two or more non-empty
        buckets an entry of an empty bucket goes to every rank), each rank computes its part of the witness
        (b200_dstate_sharded_witness), and one all_gather_object of the partial dicts, or of a rank's error, is merged.  A
        call that fails on one rank after the frontier is read raises StateRootError on every rank, so no rank is left
        waiting in an exchange.  At world > 1 a torch.distributed process group must be initialised, also when the object
        was made with `comm`."""
        from .engine import _witness_mode
        _witness_mode(mode)                                            # a bad mode: ValueError on every rank alike
        for k in post.storages:
            if k not in post.accounts:
                raise StateRootError(f"missing account {k.hex()}")
        ds = self.local.ds
        part = lambda keep: HashedPostState({k: a for k, a in post.accounts.items() if keep(k)},
                                            {k: s for k, s in post.storages.items() if keep(k)})
        kept, error = 0, None
        try:
            kept = ds.witness_root_kept(apply_layout(self._part(post), destroyed_slots=True)[1], mode)
        except Exception as e:  # noqa: BLE001
            error = str(e)
        extra = np.concatenate([np.array([kept], "<u2").view(np.uint8), np.array([error is not None], np.uint8)])
        merged, hash_mask, tree_mask, extras = self._gather_root_branch(extra)
        failed = [r for r in range(self.world) if extras[r, 2]]
        if failed:
            raise StateRootError(error if error is not None else f"witness: the kept pre-pass failed on rank {failed[0]}")
        root_kept = int(np.bitwise_or.reduce(extras[:, :2].copy().view("<u2")[:, 0]))
        owner = self._answering_rank(merged)
        every_rank = sum(1 for k in range(16) if merged[k, 34]) >= 2      # an entry of an empty bucket goes to every rank
        mine = lambda k: owner(k) == self.rank or (every_rank and not merged[k[0] >> 4, 34])
        block = apply_layout(part(mine), destroyed_slots=True)[1]
        whole_block_empty = not post.accounts and not post.storages
        try:
            result = ds.sharded_witness(merged, hash_mask, tree_mask, root_kept, block, mode,
                                        always_include_root_node=always_include_root_node and whole_block_empty)
        except Exception as e:  # noqa: BLE001
            result = f"rank {self.rank}: {e}"
        parts = [result]
        if self.world > 1:
            import torch.distributed as dist
            parts = [None] * self.world
            dist.all_gather_object(parts, result, group=self.group)
        errors = [p for p in parts if isinstance(p, str)]
        if errors:
            raise StateRootError(errors[0])
        out = {}
        for p in parts:
            out.update(p)
        return out

    def close(self):
        self.local.close()


def list_range_of(rank: int, world: int, n_lists: int) -> Tuple[int, int]:
    """Contiguous share of a batch of lists (blocks) for a rank."""
    return rank * n_lists // world, (rank + 1) * n_lists // world


def sharded_ordered_trie_roots(engine: Engine, lists, rank: int, world: int, group=None):
    """Ordered (transactions / receipts / withdrawals) roots of a batch of lists over `world` ranks: the lists are
    independent tries, so rank r folds lists [r·n/world, (r+1)·n/world) with b200_ordered_roots — no data-path
    collective — and only the 32-byte roots are all-gathered.  `lists` may be the full batch on every rank (only the
    rank's share is read).  -> all roots, in list order, on every rank."""
    from .ordered_root import ordered_trie_roots
    n = len(lists)
    lo, hi = list_range_of(rank, world, n)
    mine = ordered_trie_roots(engine, lists[lo:hi])
    if world == 1:
        return mine
    import torch
    import torch.distributed as dist
    width = (n + world - 1) // world                                   # every rank contributes a fixed-size block
    buf = np.zeros((width, 32), np.uint8)
    if mine:
        buf[:len(mine)] = np.frombuffer(b"".join(mine), np.uint8).reshape(-1, 32)
    dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
    t = torch.from_numpy(buf.reshape(-1)).to(dev)
    gathered = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(gathered, t, group=group)
    out = []
    for r in range(world):
        r_lo, r_hi = list_range_of(r, world, n)
        rows = gathered[r].cpu().numpy().reshape(width, 32)
        out += [rows[i].tobytes() for i in range(r_hi - r_lo)]
    return out

"""Host-side mirror of reth's ordered-root interface (crates/trie/common/src/ordered_root.rs) over the GPU engine.

`OrderedTrieRootEncodedBuilder` keeps the reference's names, argument meaning and error behaviour (:146-257,
`OrderedRootError` :9-80).  The reference flushes items into a HashBuilder as soon as the key order allows; here items
are only buffered — the trie of a list is built in one `b200_ordered_roots` call at `finalize()`, and
`ordered_trie_roots` folds the lists of many blocks (transactions, receipts, withdrawals of a batch of blocks during
pipeline sync) in a single call, which is where the device pays off.  There is no CPU path: without the CUDA library
`Engine` raises.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import numpy as np

from .engine import Engine

EMPTY_ROOT_HASH = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")


class OrderedRootError(Exception):
    """ordered_root.rs:9-80.  kind is one of "Incomplete", "IndexOutOfBounds", "DuplicateIndex"."""

    def __init__(self, kind: str, **fields):
        self.kind, self.fields = kind, fields
        if kind == "Incomplete":
            msg = f"incomplete: expected {fields['expected']} items, received {fields['received']}"
        elif kind == "IndexOutOfBounds":
            msg = f"index {fields['index']} out of bounds for length {fields['len']}"
        else:
            msg = f"duplicate item at index {fields['index']}"
        super().__init__(msg)

    def is_incomplete(self) -> bool:
        return self.kind == "Incomplete"

    def is_index_out_of_bounds(self) -> bool:
        return self.kind == "IndexOutOfBounds"

    def is_duplicate_index(self) -> bool:
        return self.kind == "DuplicateIndex"

    def index(self) -> Optional[int]:
        return self.fields.get("index")

    def __eq__(self, other):
        return isinstance(other, OrderedRootError) and (self.kind, self.fields) == (other.kind, other.fields)

    __hash__ = Exception.__hash__


def pack_lists(lists: Sequence[Sequence[bytes]]):
    """[[item bytes, ...], ...] -> (values u8, value_offsets u64 [n+1], seg_offsets u64 [n_lists+1])."""
    items = [it for l in lists for it in l]
    value_offsets = np.zeros(len(items) + 1, np.uint64)
    if items:
        value_offsets[1:] = np.cumsum([len(it) for it in items], dtype=np.uint64)
    seg_offsets = np.zeros(len(lists) + 1, np.uint64)
    if len(lists):
        seg_offsets[1:] = np.cumsum([len(l) for l in lists], dtype=np.uint64)
    values = np.frombuffer(b"".join(items), np.uint8) if items else np.zeros(0, np.uint8)
    return values, value_offsets, seg_offsets


def ordered_trie_roots(engine: Engine, lists: Sequence[Sequence[bytes]]) -> List[bytes]:
    """Roots of many lists of pre-encoded items in one device call (alloy_trie::root::ordered_trie_root_encoded each)."""
    if not len(lists):
        return []
    roots = engine.ordered_roots(*pack_lists(lists))
    return [r.tobytes() for r in roots]


def ordered_trie_root_encoded(engine: Engine, items: Iterable[bytes]) -> bytes:
    """alloy_trie::root::ordered_trie_root_encoded — what calculate_transaction_root / calculate_receipt_root /
    calculate_withdrawals_root return for the items' EIP-2718 encodings."""
    return engine.ordered_root(list(items))


class OrderedTrieRootEncodedBuilder:
    """ordered_root.rs:131-257.  Items may be pushed in any order by index; `finalize` needs all of them."""

    def __init__(self, engine: Engine, len: int):  # noqa: A002 (the reference's parameter name)
        self.engine = engine
        self.len = int(len)
        self.received = 0
        self.pending: List[Optional[bytes]] = [None] * self.len

    @classmethod
    def new(cls, engine: Engine, len: int) -> "OrderedTrieRootEncodedBuilder":  # noqa: A002
        return cls(engine, len)

    def push(self, index: int, data: bytes) -> None:
        if index >= self.len or index < 0:
            raise OrderedRootError("IndexOutOfBounds", index=index, len=self.len)
        if self.pending[index] is not None:
            raise OrderedRootError("DuplicateIndex", index=index)
        self.push_unchecked(index, data)

    def push_unchecked(self, index: int, data: bytes) -> None:
        self.pending[index] = bytes(data)
        self.received += 1

    def is_complete(self) -> bool:
        return self.received == self.len

    def pushed_count(self) -> int:
        return self.received

    def expected_count(self) -> int:
        return self.len

    def finalize(self) -> bytes:
        if self.len == 0:
            return EMPTY_ROOT_HASH
        if self.received != self.len:
            raise OrderedRootError("Incomplete", expected=self.len, received=self.received)
        return self.engine.ordered_root(self.pending)

"""Engine — thin Python handle on a b200_ctx (one per GPU / per process).

numpy arrays go through the host-pointer entry points (H2D + compute + D2H inside the call: the e2e path);
torch CUDA tensors go through the *_dev entry points (inputs resident in HBM, asynchronous on the ctx stream).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import B200Error, FrontierEntry, Proofs, Stats, Updates, Witness

ACCOUNT_DTYPE = np.dtype([("nonce", "<u8"), ("balance", "u1", (32,)), ("code_hash", "u1", (32,))])
KECCAK_EMPTY = bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")
EMPTY_ROOT_HASH = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")


def _np(a, dtype=np.uint8):
    return np.ascontiguousarray(a, dtype=dtype)


def _ptr(a):
    return None if a is None else a.ctypes.data


def _out_array(a, shape, dtype):
    """A result array: the caller's (checked: shape, dtype, C-contiguous, writeable) or a fresh one."""
    if a is None:
        return np.empty(shape, dtype)
    if not isinstance(a, np.ndarray) or a.shape != tuple(shape) or a.dtype != np.dtype(dtype) \
            or not a.flags.c_contiguous or not a.flags.writeable:
        raise B200Error(_lib.ERR_INVALID_ARG, f"result array must be a writeable C-contiguous {np.dtype(dtype)}{tuple(shape)}")
    return a


def _unpack_nibbles(packed: bytes, n: int) -> bytes:
    return bytes(x for b in packed for x in (b >> 4, b & 15))[:n]


def _pack_paths(paths) -> tuple:
    """nibble paths -> (lengths u8[n], [n][32] packed high-first, zero padded): the path layout of b200_updates"""
    n = len(paths)
    lens = np.array([len(p) for p in paths], np.uint8)
    packed = np.zeros((n, 32), np.uint8)
    for i, p in enumerate(paths):
        nib = bytes(p) + b"\0" * (len(p) & 1)
        packed[i, :len(nib) // 2] = np.frombuffer(bytes(nib[k] << 4 | nib[k + 1] for k in range(0, len(nib), 2)), np.uint8)
    return lens, packed


def updates_to_records(u: Updates, lib, sort: bool = True) -> list:
    """-> [(trie_id, path_nibbles, state_mask, tree_mask, hash_mask, [hashes])] sorted by (trie_id, path);
    releases the library-owned buffers.  (sort=False keeps the library's order: full builds already deliver table
    order, dirty subsets do not.)"""
    n = int(u.n_nodes)
    res = []
    if n:
        tid = np.ctypeslib.as_array(u.trie_id, (n,))
        pl = np.ctypeslib.as_array(u.path_len, (n,))
        pp = np.ctypeslib.as_array(u.path_packed, (n, 32))
        sm = np.ctypeslib.as_array(u.state_mask, (n,))
        tm = np.ctypeslib.as_array(u.tree_mask, (n,))
        hm = np.ctypeslib.as_array(u.hash_mask, (n,))
        ho = np.ctypeslib.as_array(u.hash_offset, (n + 1,))
        nh = int(ho[n])
        hs = np.ctypeslib.as_array(u.hashes, (max(nh, 1), 32))
        for i in range(n):
            res.append((int(tid[i]), _unpack_nibbles(pp[i].tobytes(), int(pl[i])), int(sm[i]), int(tm[i]),
                        int(hm[i]), [hs[j].tobytes() for j in range(int(ho[i]), int(ho[i + 1]))]))
    lib.b200_updates_release(C.byref(u))
    if sort:
        res.sort(key=lambda r: (r[0], r[1]))
    return res


class Engine:
    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        if self.lib.b200_device_count() <= 0:
            raise B200Error(_lib.ERR_NO_DEVICE, "no CUDA device: reth_b200 has no CPU path")
        self.ctx = self.lib.b200_create(device)
        if not self.ctx:
            raise B200Error(self.lib.b200_create_status(), f"b200_create({device}) failed")
        self.device = device
        self._pinned = []

    def close(self):
        if getattr(self, "ctx", None):
            self.lib.b200_destroy(self.ctx)
            self.ctx = None
            for p in self._pinned:
                self.lib.b200_host_free(p)
            self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise B200Error(rc, self.lib.b200_last_error(self.ctx).decode())

    # ------------------------------------------------------------------ plumbing
    def version(self) -> str:
        return self.lib.b200_version().decode()

    def set_stream(self, cuda_stream: int | None):
        """cuda_stream: a cudaStream_t handle (0 = legacy default stream); None = the context's own stream."""
        handle = C.c_void_p(-1) if cuda_stream is None else C.c_void_p(cuda_stream)
        self._check(self.lib.b200_set_stream(self.ctx, handle))

    def use_torch_stream(self):
        import torch
        self.set_stream(torch.cuda.current_stream(self.device).cuda_stream)

    def sync(self):
        self._check(self.lib.b200_sync(self.ctx))

    def launch_count(self) -> int:
        return int(self.lib.b200_launch_count(self.ctx))

    def device_bytes(self) -> int:
        return int(self.lib.b200_device_bytes(self.ctx))

    def last_stats(self) -> dict:
        s = Stats()
        self._check(self.lib.b200_last_stats(self.ctx, C.byref(s)))
        return s.as_dict()

    def pinned_empty(self, shape, dtype=np.uint8) -> np.ndarray:
        """numpy array over page-locked memory from b200_host_alloc; released by close()."""
        count = int(np.prod(shape))
        nbytes = max(count * np.dtype(dtype).itemsize, 1)
        p = self.lib.b200_host_alloc(nbytes)
        if not p:
            raise B200Error(_lib.ERR_OOM, "b200_host_alloc failed")
        self._pinned.append(p)
        buf = (C.c_uint8 * nbytes).from_address(p)
        return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)

    # ------------------------------------------------------------------ keccak
    def keccak256_fixed(self, msgs: np.ndarray, msg_len: int | None = None, out: np.ndarray | None = None) -> np.ndarray:
        """msgs: uint8[n, stride]; digest of the first msg_len bytes of every row -> uint8[n, 32]."""
        if msgs.dtype != np.uint8 or msgs.ndim != 2 or not msgs.flags.c_contiguous:
            msgs = _np(msgs)
        n, stride = msgs.shape
        if out is None:
            out = np.empty((n, 32), np.uint8)
        self._check(self.lib.b200_keccak256_fixed(self.ctx, _ptr(msgs), msg_len or stride, stride, n, _ptr(out)))
        return out

    def keccak256_var(self, data: np.ndarray, offsets: np.ndarray) -> np.ndarray:
        data = _np(data)
        offsets = _np(offsets, np.uint64)
        n = len(offsets) - 1
        out = np.empty((n, 32), np.uint8)
        self._check(self.lib.b200_keccak256_var(self.ctx, _ptr(data), _ptr(offsets), n, _ptr(out)))
        return out

    def keccak256(self, data: bytes) -> bytes:
        d = np.frombuffer(bytes(data) or b"\0", np.uint8)
        return self.keccak256_var(d, np.array([0, len(data)], np.uint64))[0].tobytes()

    def hash_sort_keys(self, msgs: np.ndarray, msg_len: int | None = None, out=None, perm=None):
        """-> (sorted digests uint8[n,32], perm uint32[n]): digest[perm[i]] is the i-th smallest.  `out` / `perm`: the
        caller's result arrays (page-locked ones from pinned_empty make the read-back a plain DMA)."""
        msgs = _np(msgs)
        n, stride = msgs.shape
        out = _out_array(out, (n, 32), np.uint8)
        perm = _out_array(perm, (n,), np.uint32)
        self._check(self.lib.b200_hash_sort_keys(self.ctx, _ptr(msgs), msg_len or stride, stride, n, _ptr(out), _ptr(perm)))
        return out, perm

    def hash_sort_storage(self, addresses: np.ndarray, addr_index: np.ndarray, slots: np.ndarray, out=None, perm=None):
        """StorageHashing full pass: entry i = (addresses[addr_index[i]], slots[i]) -> (composite keys uint8[n,64]
        sorted ascending, perm uint32[n]).  `out` / `perm` as in hash_sort_keys."""
        addresses = _np(addresses).reshape(-1, 20)
        addr_index = _np(addr_index, np.uint32)
        slots = _np(slots).reshape(-1, 32)
        n = len(slots)
        out = _out_array(out, (n, 64), np.uint8)
        perm = _out_array(perm, (n,), np.uint32)
        self._check(self.lib.b200_hash_sort_storage(self.ctx, _ptr(addresses), len(addresses), _ptr(addr_index),
                                                    _ptr(slots), n, _ptr(out), _ptr(perm)))
        return out, perm

    def root_from_items(self, keys, key_nibbles, item_flags, values, storage_roots32, seg_offsets, account: bool,
                        want_updates: bool = False):
        """b200_root_from_items: the fold of an incremental run over leaves (key_nibbles == 64) and stored hashes of unchanged
        subtrees (key_nibbles = path length).  -> roots uint8[tries, 32] [, records]."""
        keys = _np(keys).reshape(-1, 32)
        n = len(keys)
        key_nibbles, item_flags = _np(key_nibbles), _np(item_flags)
        values = _np(values).reshape(n, 72 if account else 32)
        sr = None if storage_roots32 is None else _np(storage_roots32).reshape(n, 32)
        so = None if seg_offsets is None else _np(seg_offsets, np.uint64)
        if len(key_nibbles) != n or len(item_flags) != n:
            raise ValueError("one key_nibbles / item_flags entry per item")
        if so is not None and (int(so[0]) != 0 or int(so[-1]) != n):
            raise ValueError("seg_offsets must start at 0 and end at the number of items")
        tries = 1 if so is None else len(so) - 1
        roots = np.empty((max(tries, 1), 32), np.uint8)
        u, s = Updates(), Stats()
        self._check(self.lib.b200_root_from_items(self.ctx, _ptr(keys), _ptr(key_nibbles), _ptr(item_flags), _ptr(values), _ptr(sr),
                                                  _ptr(so), tries if so is not None else 0, n, 1 if account else 0, _ptr(roots),
                                                  C.byref(u) if want_updates else None, C.byref(s)))
        roots = roots[:tries]
        if want_updates:
            return roots, updates_to_records(u, self.lib)
        return roots

    def witness_roots(self, parent_roots, witnesses, blocks):
        """b200_witness_roots: the post-block state root of every block from its parent root, its execution witness and the
        block alone.  witnesses[b]: a list of node RLPs or a {hash: rlp} dict (only the RLPs are sent); blocks[b]: the
        `DynamicState.apply` array tuple (acct_keys, accounts, flags, slot_keys, values, seg_offsets).
        -> (roots uint8[n, 32], statuses int32[n]): per block OK, ERR_WITNESS_INCOMPLETE or ERR_INVALID_ARG (root zeroed)."""
        args = witness_batch_arrays(parent_roots, witnesses, blocks)
        n = args[0]
        roots = np.zeros((n, 32), np.uint8)
        status = np.zeros(n, np.int32)
        s = Stats()
        self._check(self.lib.b200_witness_roots(self.ctx, n, *(_ptr(a) for a in args[1:]), _ptr(roots), _ptr(status), C.byref(s)))
        return roots, status

    def hash_changesets(self, acct_addresses, storage_addresses, storage_slots) -> dict:
        """b200_hash_changesets: the account / storage changesets of a block range (addresses uint8[na,20]; rows
        (address uint8[ns,20], slot uint8[ns,32]) in changeset order) -> the range's dirty set: unique hashed keys sorted,
        the index of the first (oldest) entry of each, the storage CSR and the account prefix set."""
        from ._lib import ChangesetHashes
        a = _np(acct_addresses).reshape(-1, 20)
        sa = _np(storage_addresses).reshape(-1, 20)
        ss = _np(storage_slots).reshape(-1, 32)
        if len(sa) != len(ss):
            raise ValueError("storage changeset rows need one address and one slot each")
        o = ChangesetHashes()
        self._check(self.lib.b200_hash_changesets(self.ctx, _ptr(a), len(a), _ptr(sa), _ptr(ss), len(ss), C.byref(o)))
        arr = lambda p, shape, n: np.ctypeslib.as_array(p, shape).copy() if n else np.zeros(shape, np.uint8 if len(shape) == 2 else None)
        na, nsa, nl, npx = int(o.n_accounts), int(o.n_storage_accounts), int(o.n_slots), int(o.n_prefix)
        res = {
            "account_keys": arr(o.account_keys32, (na, 32), na),
            "account_first": np.ctypeslib.as_array(o.account_first, (na,)).copy() if na else np.zeros(0, np.uint32),
            "storage_account_keys": arr(o.storage_account_keys32, (nsa, 32), nsa),
            "storage_seg_offsets": np.ctypeslib.as_array(o.storage_seg_offsets, (nsa + 1,)).copy(),
            "slot_keys": arr(o.slot_keys32, (nl, 32), nl),
            "slot_first": np.ctypeslib.as_array(o.slot_first, (nl,)).copy() if nl else np.zeros(0, np.uint32),
            "account_prefix_keys": arr(o.account_prefix_keys32, (npx, 32), npx),
        }
        self.lib.b200_changeset_hashes_release(C.byref(o))
        return res

    # device-resident (torch) variants ------------------------------------------------------------
    def keccak256_fixed_dev(self, t_in, msg_len: int, stride: int, n: int, t_out):
        self._check(self.lib.b200_keccak256_fixed_dev(self.ctx, t_in.data_ptr(), msg_len, stride, n, t_out.data_ptr()))

    def hash_sort_keys_dev(self, t_in, msg_len: int, stride: int, n: int, t_sorted, t_perm):
        self._check(self.lib.b200_hash_sort_keys_dev(self.ctx, t_in.data_ptr(), msg_len, stride, n,
                                                     t_sorted.data_ptr(), t_perm.data_ptr()))

    def hash_sort_storage_dev(self, t_addresses, n_addr: int, t_addr_index, t_slots, n: int, t_sorted64, t_perm):
        self._check(self.lib.b200_hash_sort_storage_dev(self.ctx, t_addresses.data_ptr(), n_addr, t_addr_index.data_ptr(),
                                                        t_slots.data_ptr(), n, t_sorted64.data_ptr(), t_perm.data_ptr()))

    def sort_keys32_dev(self, t_keys, n: int, t_sorted, t_perm):
        self._check(self.lib.b200_sort_keys32_dev(self.ctx, t_keys.data_ptr(), n, t_sorted.data_ptr(), t_perm.data_ptr()))

    # ------------------------------------------------------------------ roots (host buffers)
    def storage_roots(self, slot_keys, values, seg_offsets, want_updates=False, want_stats=False):
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        _check_segments(seg_offsets, len(slot_keys), len(values))
        m = len(seg_offsets) - 1
        roots = np.empty((m, 32), np.uint8)
        u, s = Updates(), Stats()
        self._check(self.lib.b200_storage_roots(self.ctx, _ptr(slot_keys), _ptr(values), _ptr(seg_offsets), m,
                                                _ptr(roots), C.byref(u) if want_updates else None, C.byref(s)))
        res = [roots]
        if want_updates:
            res.append(updates_to_records(u, self.lib))
        if want_stats:
            res.append(s.as_dict())
        return res[0] if len(res) == 1 else tuple(res)

    def ordered_roots(self, values, value_offsets, seg_offsets, want_stats=False):
        """Transactions / receipts / withdrawals roots of a batch of lists of pre-encoded items — what
        OrderedTrieRootEncodedBuilder::finalize returns per list (crates/trie/common/src/ordered_root.rs:240-257).
        List l = items seg_offsets[l] .. seg_offsets[l+1] in list order; item i = values[value_offsets[i] ..
        value_offsets[i+1]).  -> roots [n_lists][32]."""
        values = _np(values).reshape(-1)
        value_offsets = _np(value_offsets, np.uint64)
        seg_offsets = _np(seg_offsets, np.uint64)
        m = len(seg_offsets) - 1
        if m < 0 or len(value_offsets) < 1:
            raise ValueError("seg_offsets / value_offsets need at least one entry")
        if int(seg_offsets[-1]) != len(value_offsets) - 1:
            raise ValueError("value_offsets must have seg_offsets[-1] + 1 entries")
        if int(value_offsets[-1]) > len(values):
            raise ValueError("value_offsets run past the end of values")
        roots = np.empty((m, 32), np.uint8)
        s = Stats()
        self._check(self.lib.b200_ordered_roots(self.ctx, _ptr(values) if len(values) else None, _ptr(value_offsets),
                                                _ptr(seg_offsets), m, _ptr(roots), C.byref(s)))
        return (roots, s.as_dict()) if want_stats else roots

    def ordered_root(self, items, want_stats=False):
        """Root of one list of pre-encoded items (bytes objects) — calculate_transaction_root / calculate_receipt_root /
        calculate_withdrawals_root over their EIP-2718 encodings."""
        items = list(items)
        value_offsets = np.zeros(len(items) + 1, np.uint64)
        if items:
            value_offsets[1:] = np.cumsum([len(it) for it in items], dtype=np.uint64)
        values = np.frombuffer(b"".join(items), np.uint8) if items else np.zeros(0, np.uint8)
        r = self.ordered_roots(values, value_offsets, np.array([0, len(items)], np.uint64), want_stats=want_stats)
        return (r[0][0].tobytes(), r[1]) if want_stats else r[0].tobytes()

    def state_root(self, acct_keys, accounts, storage_roots32=None, want_updates=False, want_stats=False):
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        sr = None if storage_roots32 is None else _np(storage_roots32).reshape(-1, 32)
        root = np.empty(32, np.uint8)
        u, s = Updates(), Stats()
        self._check(self.lib.b200_state_root(self.ctx, _ptr(acct_keys), _ptr(accounts), _ptr(sr), len(acct_keys),
                                             _ptr(root), C.byref(u) if want_updates else None, C.byref(s)))
        res = [root.tobytes()]
        if want_updates:
            res.append(updates_to_records(u, self.lib))
        if want_stats:
            res.append(s.as_dict())
        return res[0] if len(res) == 1 else tuple(res)

    def state_root_full(self, acct_keys, accounts, slot_keys, values, seg_offsets, want_updates=False,
                        want_stats=False):
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        if len(seg_offsets) != len(acct_keys) + 1:
            raise ValueError("seg_offsets must have n_accounts+1 entries")
        _check_segments(seg_offsets, len(slot_keys), len(values))
        root = np.empty(32, np.uint8)
        ua, us, s = Updates(), Updates(), Stats()
        self._check(self.lib.b200_state_root_full(
            self.ctx, _ptr(acct_keys), _ptr(accounts), len(acct_keys), _ptr(slot_keys), _ptr(values),
            _ptr(seg_offsets), _ptr(root), C.byref(ua) if want_updates else None,
            C.byref(us) if want_updates else None, C.byref(s)))
        res = [root.tobytes()]
        if want_updates:
            res += [updates_to_records(ua, self.lib), updates_to_records(us, self.lib)]
        if want_stats:
            res.append(s.as_dict())
        return res[0] if len(res) == 1 else tuple(res)

    def state_root_full_rows(self, acct_keys, accounts, slot_keys, values, seg_offsets, key_format: int = 0,
                             encode_on_host: bool = False):
        """state_root_full, with the stored nodes returned as AccountsTrie / StoragesTrie table rows in MDBX key
        order (reth_b200.tables.TableRows; key_format 0 = legacy nibble keys, 1 = storage-v2 packed keys) — what
        MerkleStage hands to write_trie_updates_sorted (crates/stages/stages/src/stages/merkle.rs:184-366).
        Rows are encoded on the device (b200_state_root_full_rows); encode_on_host=True takes the records and lays the
        rows out with b200_account_trie_rows / b200_storage_trie_rows instead (same bytes)."""
        from . import tables
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        if len(seg_offsets) != len(acct_keys) + 1:
            raise ValueError("seg_offsets must have n_accounts+1 entries")
        root = np.empty(32, np.uint8)
        if not encode_on_host:
            ra, rs = _lib.Rows(), _lib.Rows()
            self._check(self.lib.b200_state_root_full_rows(
                self.ctx, _ptr(acct_keys), _ptr(accounts), len(acct_keys), _ptr(slot_keys), _ptr(values),
                _ptr(seg_offsets), key_format, _ptr(root), C.byref(ra), C.byref(rs), None))
            return root.tobytes(), tables.TableRows(ra, self.lib), tables.TableRows(rs, self.lib)
        ua, us, s = Updates(), Updates(), Stats()
        self._check(self.lib.b200_state_root_full(
            self.ctx, _ptr(acct_keys), _ptr(accounts), len(acct_keys), _ptr(slot_keys), _ptr(values),
            _ptr(seg_offsets), _ptr(root), C.byref(ua), C.byref(us), C.byref(s)))
        try:
            arows, srows = tables.rows_from_updates(ua, us, acct_keys, key_format)
        finally:
            self.lib.b200_updates_release(C.byref(ua))
            self.lib.b200_updates_release(C.byref(us))
        return root.tobytes(), arows, srows

    def subtrie_frontier(self, acct_keys, accounts, slot_keys, values, seg_offsets) -> np.ndarray:
        """This rank's 16-entry frontier as uint8[16, 68] (b200_frontier_entry records)."""
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        fr = (FrontierEntry * 16)()
        s = Stats()
        self._check(self.lib.b200_subtrie_frontier(self.ctx, _ptr(acct_keys), _ptr(accounts), len(acct_keys),
                                                   _ptr(slot_keys), _ptr(values), _ptr(seg_offsets), fr, C.byref(s)))
        return np.frombuffer(bytes(fr), np.uint8).reshape(16, 68).copy()

    def root_from_frontier(self, frontier: np.ndarray) -> bytes:
        frontier = _np(frontier).reshape(16, 68)
        fr = (FrontierEntry * 16).from_buffer_copy(frontier.tobytes())
        root = np.empty(32, np.uint8)
        self._check(self.lib.b200_root_from_frontier(self.ctx, fr, _ptr(root)))
        return root.tobytes()

    # ------------------------------------------------------------------ roots (device buffers, torch tensors)
    def storage_roots_dev(self, t_keys, t_vals, t_offs, n_accounts: int, n_slots: int, t_roots):
        self._check(self.lib.b200_storage_roots_dev(self.ctx, t_keys.data_ptr(), t_vals.data_ptr(), t_offs.data_ptr(),
                                                    n_accounts, n_slots, t_roots.data_ptr()))

    def ordered_roots_dev(self, t_values, t_value_offsets, t_seg_offsets, n_lists: int, n_items: int, t_roots):
        self._check(self.lib.b200_ordered_roots_dev(self.ctx, t_values.data_ptr(), t_values.numel() * t_values.element_size(),
                                                    t_value_offsets.data_ptr(), t_seg_offsets.data_ptr(), n_lists, n_items,
                                                    t_roots.data_ptr()))

    def state_root_dev(self, t_keys, t_accts, t_sroots, n: int, t_root):
        self._check(self.lib.b200_state_root_dev(self.ctx, t_keys.data_ptr(), t_accts.data_ptr(),
                                                 t_sroots.data_ptr() if t_sroots is not None else None, n,
                                                 t_root.data_ptr()))

    def state_root_full_dev(self, t_akeys, t_accts, n_accounts: int, t_skeys, t_svals, t_offs, n_slots: int, t_root):
        self._check(self.lib.b200_state_root_full_dev(self.ctx, t_akeys.data_ptr(), t_accts.data_ptr(), n_accounts,
                                                      t_skeys.data_ptr(), t_svals.data_ptr(), t_offs.data_ptr(),
                                                      n_slots, t_root.data_ptr()))

    def subtrie_frontier_dev(self, t_akeys, t_accts, n_accounts: int, t_skeys, t_svals, t_offs, n_slots: int,
                             t_frontier):
        self._check(self.lib.b200_subtrie_frontier_dev(self.ctx, t_akeys.data_ptr(), t_accts.data_ptr(), n_accounts,
                                                       t_skeys.data_ptr(), t_svals.data_ptr(), t_offs.data_ptr(),
                                                       n_slots, t_frontier.data_ptr()))

    def root_from_frontier_dev(self, t_frontier, t_root):
        self._check(self.lib.b200_root_from_frontier_dev(self.ctx, t_frontier.data_ptr(), t_root.data_ptr()))

    def dev_status(self):
        self._check(self.lib.b200_dev_status(self.ctx))


def witness_batch_arrays(parent_roots, witnesses, blocks) -> tuple:
    """The arguments of b200_witness_roots from n_blocks .. seg_offsets, in ABI order: the parent roots, the RLPs of every
    witness concatenated (a witness is a list of node RLPs or a {hash: rlp} dict: only the RLPs are sent), and the blocks
    (`DynamicState.apply` array tuples) concatenated."""
    n = len(blocks)
    if len(parent_roots) != n or len(witnesses) != n:
        raise ValueError("one parent root and one witness per block")
    parents = _np(np.frombuffer(b"".join(bytes(p) for p in parent_roots), np.uint8) if n else np.zeros(0, np.uint8)).reshape(n, 32)
    nodes = [bytes(r) for w in witnesses for r in (w.values() if isinstance(w, dict) else w)]
    block_node = np.cumsum([0] + [len(w) for w in witnesses], dtype=np.uint64)
    rlp_off = np.cumsum([0] + [len(r) for r in nodes], dtype=np.uint64)
    rlp = np.frombuffer(b"".join(nodes) or b"\0", np.uint8)
    return (n, parents, rlp, rlp_off, block_node) + block_batch_arrays(blocks)


def _witness_mode(mode: str) -> int:
    modes = {"legacy": 0, "canonical": 1}
    if mode not in modes:
        raise ValueError(f"mode must be one of {sorted(modes)}")
    return modes[mode]


def _block_args(acct_keys, accounts, flags, slot_keys, values, seg_offsets) -> tuple:
    """One block in the `apply` layout as contiguous arrays (flags stays None when absent), its sizes checked."""
    acct_keys = _np(acct_keys).reshape(-1, 32)
    m = len(acct_keys)
    accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
    fl = None if flags is None else _np(np.asarray(flags, dtype=np.uint8))
    slot_keys = _np(slot_keys).reshape(-1, 32)
    values = _np(values).reshape(-1, 32)
    seg_offsets = _np(seg_offsets, np.uint64)
    if len(seg_offsets) != m + 1:
        raise ValueError("seg_offsets must have m+1 entries")
    if (m and int(seg_offsets[m]) != len(slot_keys)) or len(values) != len(slot_keys):
        raise ValueError("seg_offsets[m] must equal the number of slot rows (keys and values)")
    return acct_keys, accounts, fl, slot_keys, values, seg_offsets


def block_batch_arrays(blocks) -> tuple:
    """A batch of blocks (`DynamicState.apply` array tuples) concatenated, in ABI order: acct_keys, accts, acct_flags,
    block_acct_offset, slot_keys, values, seg_offsets (b200_witness_roots, b200_dstate_overlay_roots)."""
    keys, accts, flags, skeys, svals, offs, block_acct = [], [], [], [], [], [0], [0]
    for block in blocks:
        k, a, f, sk, sv, so = _block_args(*block)
        m = len(k)
        if int(so[0]) != 0 or int(so[m]) != len(sk):
            raise ValueError("seg_offsets must run from 0 to the number of slot rows")
        keys.append(k)
        accts.append(a.reshape(m))
        flags.append(np.ones(m, np.uint8) if f is None else f.reshape(m))
        skeys.append(sk)
        svals.append(sv)
        offs.extend((so[1:] + np.uint64(offs[-1])).tolist())
        block_acct.append(block_acct[-1] + m)
    cat = lambda xs, shape, dt: np.ascontiguousarray(np.concatenate(xs)) if xs else np.zeros(shape, dt)
    keys, accts, flags = cat(keys, (0, 32), np.uint8), cat(accts, 0, ACCOUNT_DTYPE), cat(flags, 0, np.uint8)
    skeys, svals = cat(skeys, (0, 32), np.uint8), cat(svals, (0, 32), np.uint8)
    return keys, accts, flags, np.array(block_acct, np.uint64), skeys, svals, np.array(offs, np.uint64)


def _prefer_bundled_nccl():
    """The library dlopens "libnccl.so.2".  In a Python host that also imports torch AFTERWARDS the system copy loaded first
    would shadow the newer one torch is linked against (same soname): point the library at the copy bundled with torch
    (nvidia-nccl wheel) when there is one and the caller has not chosen (B200_NCCL_LIB)."""
    import importlib.util
    import os
    if os.environ.get("B200_NCCL_LIB"):
        return
    try:
        spec = importlib.util.find_spec("nvidia.nccl")
        for base in (spec.submodule_search_locations or []) if spec else []:
            cand = os.path.join(base, "lib", "libnccl.so.2")
            if os.path.exists(cand):
                os.environ["B200_NCCL_LIB"] = cand
                return
    except Exception:  # noqa: BLE001 - no bundled copy: the system library is used
        pass


class Comm:
    """b200_comm_*: the NCCL communicator behind the C ABI (one rank per GPU).  `Comm.unique_id()` on rank 0, ship the 128 bytes
    to the other ranks, `Comm(engine, id, n_ranks, rank)` on every rank (collective)."""

    @staticmethod
    def unique_id() -> bytes:
        _prefer_bundled_nccl()
        buf = np.zeros(128, np.uint8)
        rc = _lib.load().b200_comm_unique_id(_ptr(buf))
        if rc != 0:
            raise B200Error(rc, "b200_comm_unique_id: NCCL not available")
        return buf.tobytes()

    def __init__(self, engine: Engine, unique_id: bytes, n_ranks: int, rank: int):
        _prefer_bundled_nccl()
        self.engine = engine
        h = C.c_void_p()
        idb = np.frombuffer(unique_id, np.uint8).copy()
        engine._check(engine.lib.b200_comm_create(engine.ctx, _ptr(idb), n_ranks, rank, C.byref(h)))
        self.handle, self.n_ranks, self.rank = h, n_ranks, rank

    def state_root_sharded(self, acct_keys, accounts, slot_keys, values, seg_offsets) -> bytes:
        """This rank's shard (whole top-nibble buckets) in, the state root out — on every rank."""
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        root = np.empty(32, np.uint8)
        s = Stats()
        self.engine._check(self.engine.lib.b200_state_root_sharded(self.handle, _ptr(acct_keys), _ptr(accounts), len(acct_keys),
                                                                   _ptr(slot_keys), _ptr(values), _ptr(seg_offsets), _ptr(root), C.byref(s)))
        return root.tobytes()

    def state_root_sharded_dev(self, t_akeys, t_accts, n_accounts: int, t_skeys, t_svals, t_offs, n_slots: int, t_root):
        self.engine._check(self.engine.lib.b200_state_root_sharded_dev(self.handle, t_akeys.data_ptr(), t_accts.data_ptr(), n_accounts,
                                                                       t_skeys.data_ptr(), t_svals.data_ptr(), t_offs.data_ptr(),
                                                                       n_slots, t_root.data_ptr()))

    def dstate_root_sharded(self, dstate) -> bytes:
        """b200_dstate_root_sharded: after every rank applied its part of a block to its shard, the state root (all ranks)."""
        root = np.empty(32, np.uint8)
        self.engine._check(self.engine.lib.b200_dstate_root_sharded(self.handle, dstate.handle, _ptr(root)))
        return root.tobytes()

    def hash_partition_dev(self, t_in, msg_len: int, stride: int, n: int, t_values, value_bytes: int, capacity: int, t_keys_out,
                           t_values_out) -> int:
        n_out = C.c_uint64(0)
        self.engine._check(self.engine.lib.b200_hash_partition_dev(
            self.handle, t_in.data_ptr(), msg_len, stride, n, t_values.data_ptr() if t_values is not None else None, value_bytes,
            capacity, t_keys_out.data_ptr(), t_values_out.data_ptr() if t_values_out is not None else None, C.byref(n_out)))
        return int(n_out.value)

    def close(self):
        if self.handle:
            self.engine.lib.b200_comm_destroy(self.handle)
            self.handle = None


class RootStream:
    """b200_root_stream_*: a state root committed in ascending account-key ranges (StateRoot::with_threshold /
    root_with_progress / with_intermediate_state, trie.rs:73-85,156; MerkleStage's chunked rebuild, merkle.rs:184-366).
    push() returns the progress and, with retain_updates, the stored nodes the range closed; finish() the root."""

    def __init__(self, engine: Engine, retain_updates: bool = False, _handle=None):
        self.engine = engine
        if _handle is None:
            h = C.c_void_p()
            engine._check(engine.lib.b200_root_stream_begin(engine.ctx, 1 if retain_updates else 0, C.byref(h)))
            _handle = h
        self.handle = _handle
        self.retain = retain_updates

    def push(self, acct_keys, accounts, slot_keys, values, seg_offsets):
        """-> progress dict [, account records (trie_id = top nibble), storage records (trie_id = account index in this push)]"""
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        n = len(acct_keys)
        if len(seg_offsets) != n + 1 or len(accounts) != n:
            raise ValueError("seg_offsets must have n_accounts + 1 entries, accounts n_accounts")
        if int(seg_offsets[0]) != 0 or int(seg_offsets[n]) != len(slot_keys) or len(values) != len(slot_keys):
            raise ValueError("seg_offsets must start at 0 and end at the number of slot rows (keys and values)")
        from ._lib import StreamProgress
        ua, us, pr = Updates(), Updates(), StreamProgress()
        w = self.retain
        self.engine._check(self.engine.lib.b200_root_stream_push(
            self.handle, _ptr(acct_keys), _ptr(accounts), n, _ptr(slot_keys), _ptr(values), _ptr(seg_offsets),
            C.byref(ua) if w else None, C.byref(us) if w else None, C.byref(pr)))
        prog = {"accounts": int(pr.accounts), "slots": int(pr.slots), "open_accounts": int(pr.open_accounts),
                "closed_buckets": int(pr.closed_buckets)}
        if not w:
            return prog
        return prog, updates_to_records(ua, self.engine.lib), updates_to_records(us, self.engine.lib)

    def finish(self):
        """-> root [, account records of the last bucket]"""
        root = np.empty(32, np.uint8)
        ua = Updates()
        self.engine._check(self.engine.lib.b200_root_stream_finish(self.handle, _ptr(root), C.byref(ua) if self.retain else None))
        if self.retain:
            return root.tobytes(), updates_to_records(ua, self.engine.lib)
        return root.tobytes()

    def checkpoint(self) -> bytes:
        """The resumable part (1104 bytes): frontier of the closed buckets + the nibble to resume from (byte 1092)."""
        from ._lib import StreamCheckpoint
        cp = StreamCheckpoint()
        self.engine._check(self.engine.lib.b200_root_stream_checkpoint(self.handle, C.byref(cp)))
        return bytes(cp)

    @staticmethod
    def resume_nibble(checkpoint: bytes) -> int:
        from ._lib import StreamCheckpoint
        return int(StreamCheckpoint.from_buffer_copy(checkpoint).resume_nibble)

    @classmethod
    def resume(cls, engine: Engine, checkpoint: bytes) -> "RootStream":
        from ._lib import StreamCheckpoint
        cp = StreamCheckpoint.from_buffer_copy(checkpoint)
        h = C.c_void_p()
        engine._check(engine.lib.b200_root_stream_resume(engine.ctx, C.byref(cp), C.byref(h)))
        return cls(engine, bool(cp.retain_updates), _handle=h)

    def close(self):
        if self.handle:
            self.engine.lib.b200_root_stream_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def _check_segments(seg_offsets, n_rows_keys: int, n_rows_values: int):
    """The C ABI takes the row count from seg_offsets[-1] and copies that many rows out of the caller's buffers: an
    inconsistent offsets array must fail here, not read past a numpy buffer."""
    if len(seg_offsets) == 0 or int(seg_offsets[0]) != 0:
        raise B200Error(_lib.ERR_INVALID_ARG, "seg_offsets must start at 0")
    if int(seg_offsets[-1]) != n_rows_keys or n_rows_values != n_rows_keys:
        raise B200Error(_lib.ERR_INVALID_ARG, "seg_offsets[-1] must equal the number of slot rows (keys and values)")


def numa_bind_thread(device: int = 0) -> int:
    """b200_numa_bind_thread: bind the calling thread (CPUs + preferred memory) to the GPU's NUMA node; -1 = no topology."""
    return int(_lib.load().b200_numa_bind_thread(int(device)))


class ResidentTrie:
    """Handle on a b200_trie: the account trie of a whole state kept in HBM for incremental roots (BASELINE config 5).
    `update` commits value changes of existing accounts by re-hashing only their root paths."""

    def __init__(self, engine: Engine, handle, root: bytes):
        self.engine, self.handle, self._root = engine, handle, root

    # -- construction
    @classmethod
    def create(cls, engine: Engine, acct_keys, accounts, storage_roots32=None) -> "ResidentTrie":
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        sr = None if storage_roots32 is None else _np(storage_roots32).reshape(-1, 32)
        h = C.c_void_p()
        root = np.empty(32, np.uint8)
        engine._check(engine.lib.b200_trie_create(engine.ctx, _ptr(acct_keys), _ptr(accounts), _ptr(sr), len(acct_keys),
                                                  C.byref(h), _ptr(root)))
        return cls(engine, h, root.tobytes())

    @classmethod
    def create_dev(cls, engine: Engine, t_keys, t_accts, t_sroots, n: int, t_root=None) -> "ResidentTrie":
        h = C.c_void_p()
        engine._check(engine.lib.b200_trie_create_dev(engine.ctx, t_keys.data_ptr(), t_accts.data_ptr(),
                                                      t_sroots.data_ptr() if t_sroots is not None else None, n,
                                                      C.byref(h), t_root.data_ptr() if t_root is not None else None))
        return cls(engine, h, b"")

    # -- updates
    def update(self, dirty_keys, new_accounts, new_storage_roots32=None, want_updates=False, want_stats=False):
        dirty_keys = _np(dirty_keys).reshape(-1, 32)
        new_accounts = np.ascontiguousarray(new_accounts, ACCOUNT_DTYPE)
        sr = None if new_storage_roots32 is None else _np(new_storage_roots32).reshape(-1, 32)
        root = np.empty(32, np.uint8)
        u, s = Updates(), Stats()
        self.engine._check(self.engine.lib.b200_trie_update(self.handle, _ptr(dirty_keys), _ptr(new_accounts), _ptr(sr),
                                                            len(dirty_keys), _ptr(root),
                                                            C.byref(u) if want_updates else None, C.byref(s)))
        self._root = root.tobytes()
        res = [self._root]
        if want_updates:
            res.append(updates_to_records(u, self.engine.lib))
        if want_stats:
            res.append(s.as_dict())
        return res[0] if len(res) == 1 else tuple(res)

    def apply(self, keys, accounts, present=None, storage_roots32=None, want_updates=False):
        """HashedPostStateSorted semantics: keys strictly ascending, present[i] False = delete.  -> (root, rebuilt[, updates])."""
        keys = _np(keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        pres = None if present is None else _np(np.asarray(present, dtype=np.uint8))
        sr = None if storage_roots32 is None else _np(storage_roots32).reshape(-1, 32)
        root = np.empty(32, np.uint8)
        rebuilt = C.c_int32(0)
        u, s = Updates(), Stats()
        self.engine._check(self.engine.lib.b200_trie_apply(self.handle, _ptr(keys), _ptr(accounts), _ptr(pres), _ptr(sr),
                                                           len(keys), _ptr(root), C.byref(rebuilt),
                                                           C.byref(u) if want_updates else None, C.byref(s)))
        self._root = root.tobytes()
        if want_updates:
            return self._root, bool(rebuilt.value), updates_to_records(u, self.engine.lib)
        return self._root, bool(rebuilt.value)

    def update_dev(self, t_keys, t_accts, t_sroots, m: int, t_root=None):
        self.engine._check(self.engine.lib.b200_trie_update_dev(
            self.handle, t_keys.data_ptr(), t_accts.data_ptr(), t_sroots.data_ptr() if t_sroots is not None else None, m,
            t_root.data_ptr() if t_root is not None else None))

    def root(self) -> bytes:
        out = np.empty(32, np.uint8)
        self.engine._check(self.engine.lib.b200_trie_root(self.handle, _ptr(out)))
        return out.tobytes()

    def device_bytes(self) -> int:
        return int(self.engine.lib.b200_trie_device_bytes(self.handle))

    def __len__(self):
        return int(self.engine.lib.b200_trie_leaves(self.handle))

    def close(self):
        if self.handle:
            self.engine.lib.b200_trie_destroy(self.handle)
            self.handle = None


class DynamicTrie:
    """Handle on a b200_dtrie: the account trie as an arena of 16-slot branch nodes in HBM; `apply` takes upserts and
    deletes in place and re-hashes only the touched paths (reth's sparse-trie role, crates/trie/sparse/src/parallel.rs).
    Validated against the oracle on the GPU (tests/test_gpu_dtrie.py) and under tools/emu."""

    def __init__(self, engine: Engine, handle, root: bytes):
        self.engine, self.handle, self._root = engine, handle, root

    @classmethod
    def create(cls, engine: Engine, acct_keys, accounts, storage_roots32=None) -> "DynamicTrie":
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        sr = None if storage_roots32 is None else _np(storage_roots32).reshape(-1, 32)
        h = C.c_void_p()
        root = np.empty(32, np.uint8)
        engine._check(engine.lib.b200_dtrie_create(engine.ctx, _ptr(acct_keys), _ptr(accounts), _ptr(sr), len(acct_keys),
                                                   C.byref(h), _ptr(root)))
        return cls(engine, h, root.tobytes())

    @classmethod
    def create_dev(cls, engine: Engine, t_keys, t_accts, t_sroots, n: int, t_root=None) -> "DynamicTrie":
        h = C.c_void_p()
        engine._check(engine.lib.b200_dtrie_create_dev(engine.ctx, t_keys.data_ptr(), t_accts.data_ptr(),
                                                       t_sroots.data_ptr() if t_sroots is not None else None, n,
                                                       C.byref(h), t_root.data_ptr() if t_root is not None else None))
        return cls(engine, h, b"")

    def apply(self, keys, accounts, present=None, storage_roots32=None, want_updates=False, want_stats=False):
        """keys strictly ascending, present[i] False = delete.  -> root [, updated records, removed paths][, stats]."""
        keys = _np(keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        pres = None if present is None else _np(np.asarray(present, dtype=np.uint8))
        sr = None if storage_roots32 is None else _np(storage_roots32).reshape(-1, 32)
        root = np.empty(32, np.uint8)
        uu, ur, s = Updates(), Updates(), Stats()
        self.engine._check(self.engine.lib.b200_dtrie_apply(self.handle, _ptr(keys), _ptr(accounts), _ptr(pres), _ptr(sr),
                                                            len(keys), _ptr(root),
                                                            C.byref(uu) if want_updates else None,
                                                            C.byref(ur) if want_updates else None, C.byref(s)))
        self._root = root.tobytes()
        res = [self._root]
        if want_updates:
            res.append(updates_to_records(uu, self.engine.lib))
            res.append([r[1] for r in updates_to_records(ur, self.engine.lib)])
        if want_stats:
            res.append(s.as_dict())
        return res[0] if len(res) == 1 else tuple(res)

    def root(self) -> bytes:
        out = np.empty(32, np.uint8)
        self.engine._check(self.engine.lib.b200_dtrie_root(self.handle, _ptr(out)))
        return out.tobytes()

    def device_bytes(self) -> int:
        return int(self.engine.lib.b200_dtrie_device_bytes(self.handle))

    def nodes(self) -> int:
        return int(self.engine.lib.b200_dtrie_nodes(self.handle))

    def __len__(self):
        return int(self.engine.lib.b200_dtrie_leaves(self.handle))

    def close(self):
        if self.handle:
            self.engine.lib.b200_dtrie_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DynamicState:
    """Handle on a b200_dstate: accounts AND all storage tries resident; `apply` commits one block's hashed post state in
    place (see include/b200trie.h).  Validated against the oracle on the GPU (tests/test_gpu_dstate.py)."""
    EXISTS, UNCHANGED, WIPED = 1, 2, 4

    def __init__(self, engine: Engine, handle, root: bytes):
        self.engine, self.handle, self._root = engine, handle, root

    @classmethod
    def create(cls, engine: Engine, acct_keys, accounts, slot_keys, values, seg_offsets, sharded: bool = False) -> "DynamicState":
        """sharded=True: one rank's shard of a state split by top key nibble (b200_dstate_create_sharded): use `frontier()`
        after every apply, gather the entries of all ranks and finish with Engine.root_from_frontier."""
        acct_keys = _np(acct_keys).reshape(-1, 32)
        accounts = np.ascontiguousarray(accounts, ACCOUNT_DTYPE)
        slot_keys = _np(slot_keys).reshape(-1, 32)
        values = _np(values).reshape(-1, 32)
        seg_offsets = _np(seg_offsets, np.uint64)
        if len(seg_offsets) != len(acct_keys) + 1:
            raise ValueError("seg_offsets must have n_accounts+1 entries")
        if int(seg_offsets[-1]) != len(slot_keys) or len(values) != len(slot_keys):
            raise ValueError("seg_offsets[-1] must equal the number of slot rows (keys and values)")
        h = C.c_void_p()
        root = np.empty(32, np.uint8)
        fn = engine.lib.b200_dstate_create_sharded if sharded else engine.lib.b200_dstate_create
        engine._check(fn(engine.ctx, _ptr(acct_keys), _ptr(accounts), len(acct_keys), _ptr(slot_keys), _ptr(values),
                         _ptr(seg_offsets), C.byref(h), _ptr(root)))
        return cls(engine, h, root.tobytes())

    @classmethod
    def create_dev(cls, engine: Engine, p_acct_keys: int, p_accts: int, n_accounts: int, p_slot_keys: int, p_values: int,
                   p_seg_offsets: int, n_slots: int, sharded: bool = False) -> "DynamicState":
        """Seed from device-resident arrays given as raw device addresses (torch tensors: `.data_ptr()`)."""
        h = C.c_void_p()
        engine._check(engine.lib.b200_dstate_create_dev(engine.ctx, p_acct_keys, p_accts, n_accounts, p_slot_keys, p_values,
                                                        p_seg_offsets, n_slots, 1 if sharded else 0, C.byref(h), None))
        ds = cls(engine, h, b"")
        ds._root = ds.root()
        return ds

    def frontier(self) -> np.ndarray:
        """(16, 68) uint8: this shard's b200_frontier_entry array as of the last apply."""
        out = (FrontierEntry * 16)()
        self.engine._check(self.engine.lib.b200_dstate_frontier(self.handle, out))
        return np.frombuffer(bytes(out), np.uint8).reshape(16, 68).copy()

    def apply(self, acct_keys, accounts, flags, slot_keys, values, seg_offsets, want_updates=False):
        """-> root, or (root, acct_updated, acct_removed_paths, storage_updated, storage_removed [(entry, path)],
        storage_deleted flags) with want_updates."""
        acct_keys, accounts, fl, slot_keys, values, seg_offsets = _block_args(acct_keys, accounts, flags, slot_keys, values, seg_offsets)
        m = len(acct_keys)
        root = np.empty(32, np.uint8)
        au, ar, su, sr, s = Updates(), Updates(), Updates(), Updates(), Stats()
        deleted = np.zeros(max(m, 1), np.uint8)
        w = want_updates
        self.engine._check(self.engine.lib.b200_dstate_apply(
            self.handle, _ptr(acct_keys), _ptr(accounts), _ptr(fl), m, _ptr(slot_keys), _ptr(values), _ptr(seg_offsets),
            _ptr(root), C.byref(au) if w else None, C.byref(ar) if w else None, C.byref(su) if w else None,
            C.byref(sr) if w else None, _ptr(deleted) if w else None, C.byref(s)))
        self._root = root.tobytes()
        if not w:
            return self._root
        lib = self.engine.lib
        return (self._root, updates_to_records(au, lib), [r[1] for r in updates_to_records(ar, lib)],
                updates_to_records(su, lib), [(r[0], r[1]) for r in updates_to_records(sr, lib)], deleted[:m].copy())

    def apply_dev(self, p_acct_keys: int, p_accts: int, p_flags, m: int, p_slot_keys: int, p_values: int, p_seg_offsets: int,
                  n_entries: int, p_root: int):
        """The block given as raw device addresses (flags may be None); the root is written to the device buffer p_root."""
        s = Stats()
        self.engine._check(self.engine.lib.b200_dstate_apply_dev(self.handle, p_acct_keys, p_accts, p_flags, m, p_slot_keys,
                                                                 p_values, p_seg_offsets, n_entries, p_root, None, None, None,
                                                                 None, None, C.byref(s)))
        return s.as_dict()

    def _take_proofs(self, p: Proofs, with_depths: bool = False, with_masks: bool = False) -> list:
        n, nn = int(p.n_targets), int(p.n_nodes)
        res = []
        if n:
            no = np.ctypeslib.as_array(p.node_offset, (n + 1,))
            ro = np.ctypeslib.as_array(p.rlp_offset, (nn + 1,))
            nd = np.ctypeslib.as_array(p.node_depth, (max(nn, 1),))
            nm = np.ctypeslib.as_array(p.node_masks, (max(nn, 1),))
            blob = np.ctypeslib.as_array(p.rlp, (max(int(ro[nn]), 1),)).tobytes()
            for t in range(n):
                rng_ = range(int(no[t]), int(no[t + 1]))
                if with_masks:
                    res.append([(int(nd[k]), blob[int(ro[k]):int(ro[k + 1])], int(nm[k])) for k in rng_])
                elif with_depths:
                    res.append([(int(nd[k]), blob[int(ro[k]):int(ro[k + 1])]) for k in rng_])
                else:
                    res.append([blob[int(ro[k]):int(ro[k + 1])] for k in rng_])
        self.engine.lib.b200_proofs_release(C.byref(p))
        return res

    def account_multiproof(self, acct_keys) -> dict:
        """MultiProof::account_subtree (crates/trie/common/src/proofs.rs): {node path (nibbles) -> RLP} over all targets,
        every node once."""
        acct_keys = _np(acct_keys).reshape(-1, 32)
        p = Proofs()
        self.engine._check(self.engine.lib.b200_dstate_account_proofs(self.handle, _ptr(acct_keys), len(acct_keys), C.byref(p)))
        out = {}
        for key, nodes in zip(acct_keys, self._take_proofs(p, with_depths=True)):
            nib = bytes(x for b in key.tobytes() for x in (b >> 4, b & 15))
            for depth, rlp in nodes:
                out[nib[:depth]] = rlp
        return out

    @staticmethod
    def _multiproof_targets(targets: dict) -> tuple:
        """MultiProofTargets in the ABI layout: (sorted addresses, account keys, slot offsets, slot keys, slot key list)."""
        addrs = sorted(targets)
        n = len(addrs)
        ak = np.frombuffer(b"".join(addrs), np.uint8).reshape(n, 32) if n else np.zeros((0, 32), np.uint8)
        slots, offs = [], [0]
        for a in addrs:
            sl = sorted(set(bytes(x) for x in targets[a]))
            slots.extend(sl)
            offs.append(len(slots))
        sk = np.frombuffer(b"".join(slots), np.uint8).reshape(len(slots), 32) if slots else np.zeros((0, 32), np.uint8)
        return addrs, ak, np.array(offs, np.uint64), sk, slots

    def _multiproof_dict(self, addrs, offs, slots, pa, sroots, ps, with_nodes: bool) -> dict:
        """The maps of multiproof() from the two b200_proofs (released here); with_nodes adds every target's raw node list
        [(node_depth, rlp, node_masks)] in order: "account_nodes"[i] and "storage_nodes"[j] (slot j over all accounts)."""
        nib = lambda k: bytes(x for b in k for x in (b >> 4, b & 15))
        out = {"account_subtree": {}, "branch_node_masks": {}, "storages": {}}
        ap = self._take_proofs(pa, with_masks=True)
        for key, nodes in zip(addrs, ap):
            kn = nib(key)
            for depth, rlp, masks in nodes:
                out["account_subtree"][kn[:depth]] = rlp
                if masks:
                    out["branch_node_masks"][kn[:depth]] = (masks >> 16, masks & 0xFFFF)
        sp = self._take_proofs(ps, with_masks=True)
        for i, a in enumerate(addrs):
            sub, bm = {}, {}
            for j in range(int(offs[i]), int(offs[i + 1])):
                kn = nib(slots[j])
                for depth, rlp, masks in sp[j]:
                    sub[kn[:depth]] = rlp
                    if masks:
                        bm[kn[:depth]] = (masks >> 16, masks & 0xFFFF)
            out["storages"][a] = {"root": sroots[i].tobytes(), "subtree": sub, "branch_node_masks": bm}
        if with_nodes:
            out["account_nodes"], out["storage_nodes"] = ap, sp
        return out

    def multiproof(self, targets: dict, with_nodes: bool = False) -> dict:
        """Proof::multiproof(MultiProofTargets) in one device call.  targets: {hashed address: iterable of hashed slots}.
        -> {"account_subtree": {path: rlp}, "branch_node_masks": {path: (hash_mask, tree_mask)},
            "storages": {address: {"root": bytes, "subtree": {path: rlp}, "branch_node_masks": {...}}}} — the maps of
        MultiProof / StorageMultiProof (crates/trie/common/src/proofs.rs:180-188,594-602); branch_node_masks holds the
        branch nodes of the proof that reth stores in its trie tables (what Proof::with_branch_node_masks(true) collects).
        with_nodes: also every target's node list, in order (see _multiproof_dict)."""
        addrs, ak, so, sk, slots = self._multiproof_targets(targets)
        n = len(addrs)
        sroots = np.zeros((max(n, 1), 32), np.uint8)
        pa, ps = Proofs(), Proofs()
        self.engine._check(self.engine.lib.b200_dstate_multiproof(self.handle, _ptr(ak), n, _ptr(so), _ptr(sk), C.byref(pa), _ptr(sroots),
                                                                  C.byref(ps)))
        return self._multiproof_dict(addrs, so, slots, pa, sroots, ps, with_nodes)

    def frontier_masks(self) -> tuple:
        """b200_dstate_frontier_masks, on a sharded state: (hash_mask, tree_mask), the bits this shard's buckets set in the
        masks of the depth-0 root branch of the whole state.  The ranks OR them."""
        h, t = C.c_uint16(), C.c_uint16()
        self.engine._check(self.engine.lib.b200_dstate_frontier_masks(self.handle, C.byref(h), C.byref(t)))
        return h.value, t.value

    def sharded_multiproof(self, merged, hash_mask: int, tree_mask: int, targets: dict, with_nodes: bool = False) -> dict:
        """b200_dstate_sharded_multiproof: multiproof(targets) of the whole state, from this shard.  merged: (16, 68) uint8,
        the owner's frontier entry of every bucket (as for Engine.root_from_frontier); hash_mask / tree_mask: the OR of every
        rank's frontier_masks().  Every target must be one this shard answers (include/b200trie.h).  -> the dict of
        multiproof(), equal to multiproof() of the same targets on an unsharded state of all accounts."""
        fr = (FrontierEntry * 16).from_buffer_copy(_np(merged).reshape(16, 68).tobytes())
        addrs, ak, so, sk, slots = self._multiproof_targets(targets)
        n = len(addrs)
        sroots = np.zeros((max(n, 1), 32), np.uint8)
        pa, ps = Proofs(), Proofs()
        self.engine._check(self.engine.lib.b200_dstate_sharded_multiproof(self.handle, fr, hash_mask, tree_mask, _ptr(ak), n, _ptr(so),
                                                                          _ptr(sk), C.byref(pa), _ptr(sroots), C.byref(ps)))
        return self._multiproof_dict(addrs, so, slots, pa, sroots, ps, with_nodes)

    def overlay_multiproof(self, block, targets: dict, with_nodes: bool = False) -> dict:
        """b200_dstate_overlay_multiproof: multiproof(targets) of the state after `block`, against the state as it is (the
        state does not change; Proof::overlay_multiproof).  block: an `apply` array tuple (acct_keys, accounts, flags,
        slot_keys, values, seg_offsets).  -> the dict of multiproof() plus "root", the root `apply(*block)` would return."""
        keys, accts, flags, _, skeys, svals, seg = block_batch_arrays([block])
        addrs, ak, so, sk, slots = self._multiproof_targets(targets)
        n = len(addrs)
        sroots = np.zeros((max(n, 1), 32), np.uint8)
        root = np.zeros(32, np.uint8)
        pa, ps, s = Proofs(), Proofs(), Stats()
        self.engine._check(self.engine.lib.b200_dstate_overlay_multiproof(
            self.handle, _ptr(keys), _ptr(accts), _ptr(flags), len(keys), _ptr(skeys), _ptr(svals), _ptr(seg), _ptr(ak), n, _ptr(so),
            _ptr(sk), _ptr(root), C.byref(pa), _ptr(sroots), C.byref(ps), C.byref(s)))
        out = self._multiproof_dict(addrs, so, slots, pa, sroots, ps, with_nodes)
        out["root"] = root.tobytes()
        return out

    def witness(self, acct_keys, accounts, flags, slot_keys, values, seg_offsets, mode: str = "legacy",
                always_include_root_node: bool = False) -> dict:
        """Execution witness of one block given in the `apply` layout, against the state as it is (the state does not
        change): {keccak(node): node RLP} (TrieWitness::compute; mode "legacy" or "canonical", see include/b200trie.h)."""
        mode_id = _witness_mode(mode)
        acct_keys, accounts, fl, slot_keys, values, seg_offsets = _block_args(acct_keys, accounts, flags, slot_keys, values, seg_offsets)
        w = Witness()
        self.engine._check(self.engine.lib.b200_dstate_witness(
            self.handle, _ptr(acct_keys), _ptr(accounts), _ptr(fl), len(acct_keys), _ptr(slot_keys), _ptr(values), _ptr(seg_offsets),
            mode_id, 1 if always_include_root_node else 0, C.byref(w)))
        return self._witness_map(w)

    def witness_root_kept(self, block, mode: str = "legacy") -> int:
        """b200_dstate_witness_root_kept, on a sharded state: the 16-bit kept mask of this shard's part of a block (an `apply`
        array tuple, entries routed by their own top nibble): bit k = bucket k still holds a leaf after the mode's removal
        phase.  The ranks OR their masks for sharded_witness."""
        mode_id = _witness_mode(mode)
        k, a, f, sk, sv, so = _block_args(*block)
        kept = C.c_uint16()
        self.engine._check(self.engine.lib.b200_dstate_witness_root_kept(self.handle, _ptr(k), _ptr(a), _ptr(f), len(k), _ptr(sk), _ptr(sv),
                                                                         _ptr(so), mode_id, C.byref(kept)))
        return kept.value

    def sharded_witness(self, merged, hash_mask: int, tree_mask: int, kept: int, block, mode: str = "legacy",
                        always_include_root_node: bool = False) -> dict:
        """b200_dstate_sharded_witness: this shard's part of the witness of a block of the whole state.  merged, hash_mask,
        tree_mask: as for sharded_multiproof; kept: the OR of every rank's witness_root_kept; block: this rank's part (an
        `apply` array tuple; every entry must be one this shard answers, include/b200trie.h).  always_include_root_node: only
        when the whole block is empty.  -> {keccak(node): node RLP}; the union over the ranks is witness() of the whole block
        on an unsharded state of all accounts."""
        mode_id = _witness_mode(mode)
        fr = (FrontierEntry * 16).from_buffer_copy(_np(merged).reshape(16, 68).tobytes())
        k, a, f, sk, sv, so = _block_args(*block)
        w, s = Witness(), Stats()
        self.engine._check(self.engine.lib.b200_dstate_sharded_witness(
            self.handle, fr, hash_mask, tree_mask, kept, _ptr(k), _ptr(a), _ptr(f), len(k), _ptr(sk), _ptr(sv), _ptr(so), mode_id,
            1 if always_include_root_node else 0, C.byref(w), C.byref(s)))
        return self._witness_map(w)

    def overlay_witness(self, overlay_block, block, mode: str = "legacy", always_include_root_node: bool = False) -> tuple:
        """b200_dstate_overlay_witness: the witness of `block` on the state after `overlay_block`, against the state as it is
        (the state does not change; StateProofProvider::witness of a MemoryOverlayStateProvider).  Both are `apply` array
        tuples (acct_keys, accounts, flags, slot_keys, values, seg_offsets).  -> (overlay root, {keccak(node): node RLP}):
        exactly what `apply(*overlay_block)` and then `witness(*block, ...)` give on a twin state."""
        mode_id = _witness_mode(mode)
        ok, oa, of, osk, osv, oso = _block_args(*overlay_block)
        k, a, f, sk, sv, so = _block_args(*block)
        root = np.zeros(32, np.uint8)
        w, s = Witness(), Stats()
        self.engine._check(self.engine.lib.b200_dstate_overlay_witness(
            self.handle, _ptr(ok), _ptr(oa), _ptr(of), len(ok), _ptr(osk), _ptr(osv), _ptr(oso), _ptr(k), _ptr(a), _ptr(f), len(k),
            _ptr(sk), _ptr(sv), _ptr(so), mode_id, 1 if always_include_root_node else 0, _ptr(root), C.byref(w), C.byref(s)))
        return root.tobytes(), self._witness_map(w)

    def _witness_map(self, w) -> dict:
        try:
            n = int(w.n)
            if not n:
                return {}
            hashes = np.ctypeslib.as_array(w.hashes32, (n * 32,)).tobytes()
            ro = np.ctypeslib.as_array(w.rlp_offset, (n + 1,))
            blob = np.ctypeslib.as_array(w.rlp, (max(int(ro[n]), 1),)).tobytes()
            return {hashes[32 * i:32 * i + 32]: blob[int(ro[i]):int(ro[i + 1])] for i in range(n)}
        finally:
            self.engine.lib.b200_witness_release(C.byref(w))

    def overlay_roots(self, blocks, want_updates: bool = False) -> list:
        """b200_dstate_overlay_roots: the root `apply` of each block alone would return, against the state as it is (the
        state does not change).  blocks: `apply` array tuples (acct_keys, accounts, flags, slot_keys, values, seg_offsets),
        siblings on the current state, not a chain.  -> a list of 32-byte roots, or with want_updates
        (b200_dstate_overlay_roots_with_updates) one tuple per block shaped as `apply(..., want_updates=True)` returns, entry
        indices local to the block."""
        args = block_batch_arrays(blocks)
        n = len(blocks)
        roots = np.zeros((max(n, 1), 32), np.uint8)
        s = Stats()
        lib = self.engine.lib
        if not want_updates:
            self.engine._check(lib.b200_dstate_overlay_roots(self.handle, n, *(_ptr(a) for a in args), _ptr(roots), C.byref(s)))
            return [roots[b].tobytes() for b in range(n)]
        block_acct = args[3]
        m = int(block_acct[n])
        au, ar, su, sr = Updates(), Updates(), Updates(), Updates()
        deleted = np.zeros(max(m, 1), np.uint8)
        self.engine._check(lib.b200_dstate_overlay_roots_with_updates(
            self.handle, n, *(_ptr(a) for a in args), _ptr(roots), C.byref(au), C.byref(ar), C.byref(su), C.byref(sr),
            _ptr(deleted), C.byref(s)))
        au, ar, su, sr = (updates_to_records(u, lib) for u in (au, ar, su, sr))
        out = []
        for b in range(n):
            lo, hi = int(block_acct[b]), int(block_acct[b + 1])
            out.append((roots[b].tobytes(), [(0,) + r[1:] for r in au if r[0] == b], [r[1] for r in ar if r[0] == b],
                        [(r[0] - lo,) + r[1:] for r in su if lo <= r[0] < hi], [(r[0] - lo, r[1]) for r in sr if lo <= r[0] < hi],
                        deleted[lo:hi].copy()))
        return out

    def overlay_frontiers(self, blocks) -> np.ndarray:
        """b200_dstate_overlay_frontiers, on a sharded state: (n, 16, 68) uint8, row b = the entries `frontier()` would return
        after `apply` of block b alone; the state does not change.  blocks: as for `overlay_roots` (this shard's part of
        each block).  The ranks gather the rows and Engine.root_from_frontier of block b's merged entries is its root."""
        args = block_batch_arrays(blocks)
        n = len(blocks)
        out = (FrontierEntry * (16 * max(n, 1)))()
        self.engine._check(self.engine.lib.b200_dstate_overlay_frontiers(self.handle, n, *(_ptr(a) for a in args), out,
                                                                         C.byref(Stats())))
        return np.frombuffer(bytes(out), np.uint8).reshape(-1, 16, 68)[:n].copy()

    def trie_changesets(self, acct_paths, storage: dict) -> tuple:
        """b200_dstate_trie_changesets: the values the changed trie nodes of a block had before it, against the state as it
        is (the state does not change; reth's compute_trie_changesets).  acct_paths: the block's changed account-trie paths
        (nibble strings), sorted; storage: {hashed address: (is_deleted, sorted changed paths)}.  -> (account records,
        storage records), records shaped as `apply(..., want_updates=True)` returns them: (trie_id, path, state_mask,
        tree_mask, hash_mask, [hashes]), all masks 0 and no hashes for None; a storage record's trie_id is the index of its
        address in sorted(storage).  Order: account records in input order; storage records by trie, then path."""
        alen, apk = _pack_paths(acct_paths)
        addrs = sorted(storage)
        n = len(addrs)
        keys = np.frombuffer(b"".join(addrs), np.uint8).reshape(n, 32) if n else np.zeros((0, 32), np.uint8)
        flags = np.array([1 if storage[a][0] else 0 for a in addrs], np.uint8)
        paths, offs = [], [0]
        for a in addrs:
            paths.extend(storage[a][1])
            offs.append(len(paths))
        slen, spk = _pack_paths(paths)
        offs = np.array(offs, np.uint64)
        au, su, s = Updates(), Updates(), Stats()
        lib = self.engine.lib
        self.engine._check(lib.b200_dstate_trie_changesets(self.handle, _ptr(alen), _ptr(apk), len(alen), _ptr(keys), _ptr(flags), n,
                                                           _ptr(offs), _ptr(slen), _ptr(spk), C.byref(au), C.byref(su), C.byref(s)))
        return updates_to_records(au, lib, sort=False), updates_to_records(su, lib, sort=False)

    def account_proofs(self, acct_keys) -> list:
        """-> for every target hashed address the list of node RLPs from the root down (Proof::account_proof)."""
        acct_keys = _np(acct_keys).reshape(-1, 32)
        p = Proofs()
        self.engine._check(self.engine.lib.b200_dstate_account_proofs(self.handle, _ptr(acct_keys), len(acct_keys), C.byref(p)))
        return self._take_proofs(p)

    def storage_proofs(self, acct_key: bytes, slot_keys):
        """-> (storage root, [proof of every hashed slot key]) of one account (Proof::storage_proof)."""
        ak = np.frombuffer(bytes(acct_key), np.uint8).copy()
        slot_keys = _np(slot_keys).reshape(-1, 32)
        sroot = np.empty(32, np.uint8)
        p = Proofs()
        self.engine._check(self.engine.lib.b200_dstate_storage_proofs(self.handle, _ptr(ak), _ptr(slot_keys), len(slot_keys),
                                                                      _ptr(sroot), C.byref(p)))
        return sroot.tobytes(), self._take_proofs(p)

    def root(self) -> bytes:
        out = np.empty(32, np.uint8)
        self.engine._check(self.engine.lib.b200_dstate_root(self.handle, _ptr(out)))
        return out.tobytes()

    def accounts(self) -> int:
        return int(self.engine.lib.b200_dstate_accounts(self.handle))

    def slots(self) -> int:
        return int(self.engine.lib.b200_dstate_slots(self.handle))

    def device_bytes(self) -> int:
        return int(self.engine.lib.b200_dstate_device_bytes(self.handle))

    def close(self):
        if self.handle:
            self.engine.lib.b200_dstate_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

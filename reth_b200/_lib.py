"""ctypes loader for libb200trie.so (the C-ABI of include/b200trie.h).

There is no CPU fallback: if the shared library is missing, or no CUDA device is usable, the error is raised
to the caller.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200trie.so")

# b200_status (include/b200trie.h)
OK, ERR_NO_DEVICE, ERR_CUDA, ERR_INVALID_ARG, ERR_UNSORTED, ERR_ZERO_VALUE, ERR_OOM, ERR_INLINE_HASH_CHILD, \
    ERR_NOT_FOUND, ERR_WITNESS_INCOMPLETE = (0, -1, -2, -3, -4, -5, -6, -7, -8, -9)


class B200Error(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"b200 status {status}: {message}")
        self.status = status


class Updates(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_uint64),
        ("trie_id", C.POINTER(C.c_uint32)),
        ("path_len", C.POINTER(C.c_uint8)),
        ("path_packed", C.POINTER(C.c_uint8)),
        ("state_mask", C.POINTER(C.c_uint16)),
        ("tree_mask", C.POINTER(C.c_uint16)),
        ("hash_mask", C.POINTER(C.c_uint16)),
        ("hash_offset", C.POINTER(C.c_uint64)),
        ("hashes", C.POINTER(C.c_uint8)),
        ("_owner", C.c_void_p),
    ]


class Rows(C.Structure):
    """b200_rows (include/b200trie.h): table rows in MDBX key order."""
    _fields_ = [
        ("n_rows", C.c_uint64),
        ("row_offset", C.POINTER(C.c_uint64)),
        ("key_len", C.POINTER(C.c_uint32)),
        ("bytes", C.POINTER(C.c_uint8)),
        ("_owner", C.c_void_p),
    ]


class Proofs(C.Structure):
    """b200_proofs (include/b200trie.h)."""
    _fields_ = [
        ("n_targets", C.c_uint64),
        ("node_offset", C.POINTER(C.c_uint64)),
        ("n_nodes", C.c_uint64),
        ("rlp_offset", C.POINTER(C.c_uint64)),
        ("rlp", C.POINTER(C.c_uint8)),
        ("node_depth", C.POINTER(C.c_uint8)),
        ("node_masks", C.POINTER(C.c_uint32)),
        ("_owner", C.c_void_p),
    ]


class Witness(C.Structure):
    """b200_witness (include/b200trie.h)."""
    _fields_ = [
        ("n", C.c_uint64),
        ("hashes32", C.POINTER(C.c_uint8)),
        ("rlp_offset", C.POINTER(C.c_uint64)),
        ("rlp", C.POINTER(C.c_uint8)),
        ("_owner", C.c_void_p),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("leaves_added", C.c_uint64),
        ("branches_added", C.c_uint64),
        ("extension_nodes", C.c_uint64),
        ("hashed_nodes", C.c_uint64),
        ("levels", C.c_uint64),
        ("device_ms", C.c_double),
        ("keccak_f", C.c_uint64),
    ]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class FrontierEntry(C.Structure):
    _fields_ = [
        ("as_child_len", C.c_uint8),
        ("as_child", C.c_uint8 * 33),
        ("as_root_len", C.c_uint8),
        ("as_root", C.c_uint8 * 33),
    ]


assert C.sizeof(FrontierEntry) == 68


class ChangesetHashes(C.Structure):
    _fields_ = [("n_accounts", C.c_uint64), ("account_keys32", C.POINTER(C.c_uint8)), ("account_first", C.POINTER(C.c_uint32)),
                ("n_storage_accounts", C.c_uint64), ("storage_account_keys32", C.POINTER(C.c_uint8)),
                ("storage_seg_offsets", C.POINTER(C.c_uint64)), ("n_slots", C.c_uint64), ("slot_keys32", C.POINTER(C.c_uint8)),
                ("slot_first", C.POINTER(C.c_uint32)), ("n_prefix", C.c_uint64), ("account_prefix_keys32", C.POINTER(C.c_uint8)),
                ("_owner", C.c_void_p)]


class StreamProgress(C.Structure):
    _fields_ = [("accounts", C.c_uint64), ("slots", C.c_uint64), ("open_accounts", C.c_uint64), ("closed_buckets", C.c_uint32)]


class StreamCheckpoint(C.Structure):
    _fields_ = [("frontier", FrontierEntry * 16), ("closed_mask", C.c_uint32), ("resume_nibble", C.c_uint32),
                ("retain_updates", C.c_uint32), ("_reserved", C.c_uint32)]


assert C.sizeof(StreamCheckpoint) == 16 * 68 + 16

_lib = None


def load():
    """Returns the loaded library; raises if libb200trie.so has not been built (python -c 'import
    __graft_entry__ as g; g.build()' or make -C reth_b200/csrc)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `make -C reth_b200/csrc` (needs nvcc). "
                          "reth_b200 has no CPU path.")
    L = C.CDLL(LIB_PATH)
    vp, i32, u32, u64 = C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64
    PU, PS = C.POINTER(Updates), C.POINTER(Stats)

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("b200_device_count", i32)
    sig("b200_create", vp, i32)
    sig("b200_create_status", i32)
    sig("b200_destroy", None, vp)
    sig("b200_last_error", C.c_char_p, vp)
    sig("b200_version", C.c_char_p)
    sig("b200_set_stream", i32, vp, vp)
    sig("b200_sync", i32, vp)
    sig("b200_numa_bind_thread", C.c_int32, C.c_int32)
    sig("b200_host_alloc", vp, C.c_size_t)
    sig("b200_host_free", None, vp)
    sig("b200_device_bytes", u64, vp)
    sig("b200_launch_count", u64, vp)
    sig("b200_keccak256_fixed", i32, vp, vp, u32, u32, u64, vp)
    sig("b200_keccak256_fixed_dev", i32, vp, vp, u32, u32, u64, vp)
    sig("b200_keccak256_var", i32, vp, vp, vp, u64, vp)
    sig("b200_keccak256_var_dev", i32, vp, vp, vp, u64, vp)
    sig("b200_hash_sort_keys", i32, vp, vp, u32, u32, u64, vp, vp)
    sig("b200_hash_sort_keys_dev", i32, vp, vp, u32, u32, u64, vp, vp)
    sig("b200_sort_keys32_dev", i32, vp, vp, u64, vp, vp)
    sig("b200_hash_sort_storage", i32, vp, vp, u32, vp, vp, u64, vp, vp)
    sig("b200_hash_sort_storage_dev", i32, vp, vp, u32, vp, vp, u64, vp, vp)
    sig("b200_updates_release", None, PU)
    sig("b200_account_trie_rows", i32, PU, i32, C.POINTER(Rows))
    sig("b200_storage_trie_rows", i32, PU, vp, u64, i32, C.POINTER(Rows))
    sig("b200_rows_release", None, C.POINTER(Rows))
    sig("b200_storage_roots", i32, vp, vp, vp, vp, u64, vp, PU, PS)
    sig("b200_state_root", i32, vp, vp, vp, vp, u64, vp, PU, PS)
    sig("b200_state_root_full", i32, vp, vp, vp, u64, vp, vp, vp, vp, PU, PU, PS)
    sig("b200_state_root_full_rows", i32, vp, vp, vp, u64, vp, vp, vp, i32, vp, C.POINTER(Rows), C.POINTER(Rows), PS)
    sig("b200_storage_roots_dev", i32, vp, vp, vp, vp, u64, u64, vp)
    sig("b200_state_root_dev", i32, vp, vp, vp, vp, u64, vp)
    sig("b200_state_root_full_dev", i32, vp, vp, vp, u64, vp, vp, vp, u64, vp)
    sig("b200_ordered_roots", i32, vp, vp, vp, vp, u64, vp, PS)
    sig("b200_ordered_roots_dev", i32, vp, vp, u64, vp, vp, u64, u64, vp)
    sig("b200_dev_status", i32, vp)
    sig("b200_last_stats", i32, vp, PS)
    sig("b200_subtrie_frontier", i32, vp, vp, vp, u64, vp, vp, vp, C.POINTER(FrontierEntry), PS)
    sig("b200_subtrie_frontier_dev", i32, vp, vp, vp, u64, vp, vp, vp, u64, vp)
    sig("b200_root_from_frontier", i32, vp, C.POINTER(FrontierEntry), vp)
    sig("b200_root_from_frontier_dev", i32, vp, vp, vp)
    sig("b200_comm_unique_id", i32, vp)
    sig("b200_comm_create", i32, vp, vp, i32, i32, C.POINTER(vp))
    sig("b200_comm_destroy", None, vp)
    sig("b200_comm_rank", i32, vp)
    sig("b200_comm_size", i32, vp)
    sig("b200_state_root_sharded", i32, vp, vp, vp, u64, vp, vp, vp, vp, PS)
    sig("b200_state_root_sharded_dev", i32, vp, vp, vp, u64, vp, vp, vp, u64, vp)
    sig("b200_dstate_root_sharded", i32, vp, vp, vp)
    sig("b200_hash_partition_dev", i32, vp, vp, C.c_uint32, C.c_uint32, u64, vp, C.c_uint32, u64, vp, vp, C.POINTER(C.c_uint64))
    sig("b200_root_from_items", i32, vp, vp, vp, vp, vp, vp, vp, u64, u64, i32, vp, PU, PS)
    sig("b200_hash_changesets", i32, vp, vp, u64, vp, vp, u64, C.POINTER(ChangesetHashes))
    sig("b200_changeset_hashes_release", None, C.POINTER(ChangesetHashes))
    sig("b200_root_stream_begin", i32, vp, i32, C.POINTER(vp))
    sig("b200_root_stream_push", i32, vp, vp, vp, u64, vp, vp, vp, PU, PU, C.POINTER(StreamProgress))
    sig("b200_root_stream_finish", i32, vp, vp, PU)
    sig("b200_root_stream_checkpoint", i32, vp, C.POINTER(StreamCheckpoint))
    sig("b200_root_stream_resume", i32, vp, C.POINTER(StreamCheckpoint), C.POINTER(vp))
    sig("b200_root_stream_free", None, vp)
    sig("b200_trie_create", i32, vp, vp, vp, vp, u64, C.POINTER(vp), vp)
    sig("b200_trie_create_dev", i32, vp, vp, vp, vp, u64, C.POINTER(vp), vp)
    sig("b200_trie_update", i32, vp, vp, vp, vp, u64, vp, PU, PS)
    sig("b200_trie_update_dev", i32, vp, vp, vp, vp, u64, vp)
    sig("b200_trie_apply", i32, vp, vp, vp, vp, vp, u64, vp, C.POINTER(i32), PU, PS)
    sig("b200_trie_root", i32, vp, vp)
    sig("b200_trie_device_bytes", u64, vp)
    sig("b200_trie_leaves", u64, vp)
    sig("b200_trie_destroy", None, vp)
    sig("b200_dtrie_create", i32, vp, vp, vp, vp, u64, C.POINTER(vp), vp)
    sig("b200_dtrie_create_dev", i32, vp, vp, vp, vp, u64, C.POINTER(vp), vp)
    sig("b200_dtrie_apply", i32, vp, vp, vp, vp, vp, u64, vp, PU, PU, PS)
    sig("b200_dtrie_root", i32, vp, vp)
    sig("b200_dtrie_leaves", u64, vp)
    sig("b200_dtrie_nodes", u64, vp)
    sig("b200_dtrie_device_bytes", u64, vp)
    sig("b200_dtrie_destroy", None, vp)
    sig("b200_dstate_create", i32, vp, vp, vp, u64, vp, vp, vp, C.POINTER(vp), vp)
    sig("b200_dstate_create_sharded", i32, vp, vp, vp, u64, vp, vp, vp, C.POINTER(vp), vp)
    sig("b200_dstate_create_dev", i32, vp, vp, vp, u64, vp, vp, vp, u64, i32, C.POINTER(vp), vp)
    sig("b200_dstate_frontier", i32, vp, C.POINTER(FrontierEntry))
    sig("b200_dstate_apply", i32, vp, vp, vp, vp, u64, vp, vp, vp, vp, PU, PU, PU, PU, vp, PS)
    sig("b200_dstate_account_proofs", i32, vp, vp, u64, C.POINTER(Proofs))
    sig("b200_dstate_storage_proofs", i32, vp, vp, vp, u64, vp, C.POINTER(Proofs))
    sig("b200_dstate_multiproof", i32, vp, vp, u64, vp, vp, C.POINTER(Proofs), vp, C.POINTER(Proofs))
    sig("b200_dstate_frontier_masks", i32, vp, C.POINTER(C.c_uint16), C.POINTER(C.c_uint16))
    sig("b200_dstate_sharded_multiproof", i32, vp, C.POINTER(FrontierEntry), C.c_uint16, C.c_uint16, vp, u64, vp, vp,
        C.POINTER(Proofs), vp, C.POINTER(Proofs))
    sig("b200_proofs_release", None, C.POINTER(Proofs))
    sig("b200_dstate_witness", i32, vp, vp, vp, vp, u64, vp, vp, vp, i32, i32, C.POINTER(Witness))
    sig("b200_witness_release", None, C.POINTER(Witness))
    sig("b200_dstate_witness_root_kept", i32, vp, vp, vp, vp, u64, vp, vp, vp, i32, C.POINTER(C.c_uint16))
    sig("b200_dstate_sharded_witness", i32, vp, C.POINTER(FrontierEntry), C.c_uint16, C.c_uint16, C.c_uint16, vp, vp, vp, u64, vp, vp, vp,
        i32, i32, C.POINTER(Witness), C.POINTER(Stats))
    sig("b200_witness_roots", i32, vp, u64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, PS)
    sig("b200_dstate_overlay_roots", i32, vp, u64, vp, vp, vp, vp, vp, vp, vp, vp, PS)
    sig("b200_dstate_overlay_frontiers", i32, vp, u64, vp, vp, vp, vp, vp, vp, vp, C.POINTER(FrontierEntry), PS)
    sig("b200_dstate_overlay_roots_with_updates", i32, vp, u64, vp, vp, vp, vp, vp, vp, vp, vp, PU, PU, PU, PU, vp, PS)
    sig("b200_dstate_overlay_multiproof", i32, vp, vp, vp, vp, u64, vp, vp, vp, vp, u64, vp, vp, vp, C.POINTER(Proofs), vp,
        C.POINTER(Proofs), PS)
    sig("b200_dstate_overlay_witness", i32, vp, vp, vp, vp, u64, vp, vp, vp, vp, vp, vp, u64, vp, vp, vp, i32, i32, vp,
        C.POINTER(Witness), PS)
    sig("b200_dstate_trie_changesets", i32, vp, vp, vp, u64, vp, vp, u64, vp, vp, vp, PU, PU, PS)
    sig("b200_dstate_apply_dev", i32, vp, vp, vp, vp, u64, vp, vp, vp, u64, vp, PU, PU, PU, PU, vp, PS)
    sig("b200_dstate_root", i32, vp, vp)
    sig("b200_dstate_accounts", u64, vp)
    sig("b200_dstate_slots", u64, vp)
    sig("b200_dstate_device_bytes", u64, vp)
    sig("b200_dstate_destroy", None, vp)
    _lib = L
    return L

"""reth_b200 — GPU state-root engine behind reth's StateRoot / StorageRoot / HashedPostState surface.

The product is libb200trie.so (hand-written sm_90a CUDA for the H100 behind the C ABI of include/b200trie.h); this
package is the host-side mirror of the reference interface used by tests and benchmarks.
"""
from ._lib import B200Error, LIB_PATH  # noqa: F401
from .engine import ACCOUNT_DTYPE, EMPTY_ROOT_HASH, KECCAK_EMPTY, DynamicState, DynamicTrie, Comm, Engine, ResidentTrie, RootStream, numa_bind_thread  # noqa: F401
from .hashed_state import (Account, HashedPostState, HashedPostStateSorted, HashedStorage,  # noqa: F401,E402
                           HashedStorageSorted, KeccakKeyHasher, PrefixSet, PrefixSetMut, TriePrefixSets,
                           TriePrefixSetsMut, unpack_nibbles)
from .stages import AccountHashingStage, MerkleStage, StageError, StorageHashingStage, Tables  # noqa: F401,E402
from .trie import (BranchNodeCompact, DynamicStateRoot, ParallelStateRoot, ResidentStateRoot, StateRoot, StateRootError, StateRootProgress,  # noqa: F401,E402
                   StorageRoot, StorageTrieUpdates, TrieUpdates, stateless_state_root, stateless_state_roots)
from .sharded import ShardedDynamicStateRoot, sharded_ordered_trie_roots  # noqa: F401,E402
from .verify import Verifier  # noqa: F401,E402
from .ordered_root import (OrderedRootError, OrderedTrieRootEncodedBuilder, ordered_trie_root_encoded,  # noqa: F401,E402
                           ordered_trie_roots)
from .walker import IncrementalStateRoot, TrieElement, walk  # noqa: F401,E402

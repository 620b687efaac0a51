// trie_kernels.cu — level-synchronous Merkle-Patricia-Trie commitment on sm_90a.
//
// Replaces the serial stack machine of alloy-trie's HashBuilder (driven by StateRoot::calculate,
// crates/trie/trie/src/trie.rs:247-309, and StorageRoot::calculate, :659-698) by a data-parallel
// formulation over the SORTED leaf array (SURVEY.md Appendix A, "data-parallel reading"):
//
//   gap g (1..n-1) sits between leaf g-1 and leaf g;  Lp[g] = common-prefix length of the two keys in
//   nibbles (0xFF at a trie boundary).  A branch node at depth d is a maximal run of depth-d gaps with no
//   shallower gap in between; its children are the leaves / deeper branches between consecutive gaps.
//   Sorting the gaps by depth therefore yields, for every level, the list of branch nodes (CSR over gaps),
//   and levels can be hashed deepest-first with one thread per node.  S[l] / E[r] map a leaf position to the
//   frontier item that currently starts / ends there, so a node finds its <=16 children in O(1).
//
// Every node is RLP-encoded into a per-thread shared-memory strip (word-transposed: conflict-free for the
// absorb loop) and hashed with a register-resident Keccak-f[1600].  A forest of tries (all storage tries of a
// block / of the whole state) is processed in the same launches: segment boundaries are just gaps with
// Lp = 0xFF.
#include "keccak_f1600.cuh"
#include "trie_kernels.h"
#include <mutex>
#include <unordered_map>

namespace b200 {

#include "tk_strip.cuh"
#include "tk_structure.cuh"
#include "tk_leaf.cuh"
#include "tk_branch.cuh"
#include "tk_warp.cuh"
#include "tk_wavefront.cuh"
#include "tk_outputs.cuh"
#include "tk_resident.cuh"
#include "tk_frontier.cuh"
#include "tk_launchers.cuh"
#include "tk_ordered.cuh"
#include "tk_items.cuh"
#include "tk_dtrie.cuh"
#include "tk_dstate.cuh"
#include "tk_proofs.cuh"
#include "tk_dtrie_launchers.cuh"
#include "tk_witness.cuh"
#include "tk_changesets.cuh"
#include "tk_stateless.cuh"
#include "tk_overlay.cuh"

}  // namespace b200

/*
 * oracle.h — CPU restatement of reth's state-commitment path.  TEST INFRASTRUCTURE ONLY.
 *
 * This library is the parity checker and the CPU baseline.  Nothing under reth_b200/ may
 * link, import or call it; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs do.
 *
 * What it restates (reference paths relative to the root of the reth checkout):
 *   - keccak256                      alloy-primitives 1.6.0 `keccak256` (external crate; Keccak-f[1600],
 *                                    rate 136, pad 0x01..0x80) called from crates/trie/common/src/key.rs:4-18
 *   - HashBuilder / RLP / hex-prefix alloy-trie 0.9.5 `HashBuilder` (external crate), restated from its
 *                                    published algorithm (SURVEY.md Appendix A); field set matches
 *                                    crates/trie/common/src/hash_builder/state.rs:15-48
 *   - storage_root / state_root      crates/trie/trie/src/trie.rs:160-330 (StateRoot::calculate),
 *                                    :615-721 (StorageRoot::calculate), :411-455 (account leaf RLP)
 *   - TrieUpdates::finalize          crates/trie/common/src/updates.rs:140-158 (drops the empty-path entry)
 *   - ParallelStateRoot              crates/trie/parallel/src/root.rs:81-221 (storage roots fan-out,
 *                                    serial account fold)
 *   - AccountHashing/StorageHashing  crates/stages/stages/src/stages/hashing_account.rs:192-211,
 *                                    hashing_storage.rs:121-148 (keccak per key in chunks of 100)
 *
 * Parity status: PINNED by the reference's own golden vectors (SURVEY.md Appendix B), see
 * tests/test_oracle_golden.py.
 */
#ifndef RETH_B200_ORACLE_H
#define RETH_B200_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- keccak */
void orc_keccak256(const uint8_t *in, size_t len, uint8_t out[32]);
/* n fixed-length messages, `threads` worker threads (chunks of 100 keys like the rayon tasks of
 * hashing_account.rs:192-203). */
void orc_keccak256_fixed(const uint8_t *in, uint32_t msg_len, uint32_t stride, uint64_t n,
                         uint8_t *out32, int threads);
void orc_keccak256_var(const uint8_t *data, const uint64_t *offsets, uint64_t n, uint8_t *out32,
                       int threads);
/* Best-effort SIMD figure for the CPU baseline (BASELINE.md §2): 8-way AVX-512 multi-buffer Keccak, msg_len <= 135.
 * Returns 1 if it ran, 0 if the CPU lacks AVX-512F (nothing written). reth itself hashes one key at a time. */
int orc_keccak256_fixed_simd(const uint8_t *in, uint32_t msg_len, uint32_t stride, uint64_t n, uint8_t *out32,
                             int threads);

/* ---------------------------------------------------------------- HashBuilder (alloy-trie restatement) */
typedef struct orc_hb orc_hb;

typedef struct {
    uint8_t path[64]; /* nibbles, one per byte */
    uint8_t path_len;
    uint16_t state_mask, tree_mask, hash_mask;
    uint8_t n_hashes;
    uint8_t hashes[16][32];
    uint8_t has_root_hash;
    uint8_t root_hash[32];
} orc_branch_node;

orc_hb *orc_hb_new(int retain_updates);
void orc_hb_free(orc_hb *);
/* keys are nibble strings (one nibble per byte, 0..15). Return 0, or -1 on ordering violation. */
int orc_hb_add_leaf(orc_hb *, const uint8_t *key, size_t key_len, const uint8_t *value, size_t vlen);
int orc_hb_add_branch(orc_hb *, const uint8_t *key, size_t key_len, const uint8_t hash[32],
                      int stored_in_database);
void orc_hb_root(orc_hb *, uint8_t out[32]);
/* updated_branch_nodes, sorted by path. Includes the empty-path entry (reth drops it later). */
size_t orc_hb_updates_len(const orc_hb *);
const orc_branch_node *orc_hb_update_at(orc_hb *, size_t i);
/* RLP of every node pushed on the stack, in creation order (for the byte-exact proof-node vectors). */
size_t orc_hb_nodes_len(const orc_hb *);
const uint8_t *orc_hb_node_at(const orc_hb *, size_t i, size_t *len);
void orc_hb_retain_nodes(orc_hb *, int on);

/* ---------------------------------------------------------------- account / value encodings */
typedef struct {
    uint64_t nonce;
    uint8_t balance_be[32];
    uint8_t code_hash[32]; /* KECCAK_EMPTY when the account has no code */
} orc_account;

/* rlp(TrieAccount{nonce,balance,storage_root,code_hash}); returns length (<=110). */
size_t orc_encode_trie_account(const orc_account *a, const uint8_t storage_root[32], uint8_t out[112]);
/* alloy_rlp::encode_fixed_size(U256) for a big-endian 32-byte value; returns length (1..33). */
size_t orc_encode_u256(const uint8_t value_be[32], uint8_t out[33]);

/* ---------------------------------------------------------------- roots (same buffers as include/b200trie.h) */
typedef struct {
    uint64_t n_nodes;
    uint32_t *trie_id;     /* storage: account index of the segment; account trie: 0 */
    uint8_t *path_len;     /* nibbles */
    uint8_t *path_packed;  /* [n][32], high nibble first, zero padded */
    uint16_t *state_mask, *tree_mask, *hash_mask;
    uint64_t *hash_offset; /* [n+1] */
    uint8_t *hashes;       /* [hash_offset[n]][32] */
} orc_updates;

void orc_updates_free(orc_updates *);

/* Storage roots of n_accounts independent tries. slot keys sorted ascending inside each segment.
 * Zero values are rejected (-2): reth never stores them (hashed_state.rs zero == deletion). */
int orc_storage_roots(const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets,
                      uint64_t n_accounts, uint8_t *roots32, orc_updates *opt_updates, int threads);

/* Account trie over sorted hashed addresses with given storage roots. */
int orc_state_root(const uint8_t *acct_keys32, const orc_account *accts, const uint8_t *storage_roots32,
                   uint64_t n, uint8_t root32[32], orc_updates *opt_updates);

/* StateRoot::calculate restated end to end: serial when threads<=1 (crates/trie/trie/src/trie.rs:160),
 * ParallelStateRoot-shaped otherwise (crates/trie/parallel/src/root.rs:81). storage updates carry
 * trie_id = account index. */
int orc_state_root_full(const uint8_t *acct_keys32, const orc_account *accts, uint64_t n_accounts,
                        const uint8_t *slot_keys32, const uint8_t *values32_be, const uint64_t *seg_offsets,
                        uint8_t root32[32], orc_updates *opt_account_updates,
                        orc_updates *opt_storage_updates, int threads);

/* Independent second implementation (recursive, yellow-paper style; plays the part `triehash` plays in
 * crates/trie/trie/src/test_utils.rs:9-49): root of sorted (key32, value bytes) pairs. */
int orc_trie_root_recursive(const uint8_t *keys32, const uint8_t *values, const uint64_t *value_offsets,
                            uint64_t n, uint8_t root32[32]);

/* Ordered (index-keyed) trie roots of n_lists lists of pre-encoded items: list l = items seg_offsets[l] ..
 * seg_offsets[l+1] in list order, item i = values[value_offsets[i] .. value_offsets[i+1])
 * (crates/trie/common/src/ordered_root.rs:202-257). */
int orc_ordered_roots(const uint8_t *values, const uint64_t *value_offsets, const uint64_t *seg_offsets,
                      uint64_t n_lists, uint8_t *roots32);

/* Structure statistics of the last orc_state_root/orc_storage_roots call on this thread. */
typedef struct {
    uint64_t leaves, branch_nodes, extension_nodes, hashed_nodes, keccak_f, rlp_bytes_hashed;
} orc_stats;
void orc_stats_reset(void);
void orc_stats_get(orc_stats *out);

#ifdef __cplusplus
}
#endif
#endif

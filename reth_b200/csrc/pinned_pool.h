// pinned_pool.h — page-locked result blocks, recycled.
//
// Every result a call hands to the host (TrieUpdates records, table rows, proofs, changeset hashes) lives in one page-locked
// block that the caller gives back with the matching b200_*_release.  cudaMallocHost / cudaFreeHost pin / unpin pages and
// synchronise the device, which for the 44 MB of a C3-shape row set costs more than the
// block update or the row encoding that fills the block.  Released blocks are therefore kept (up to B200_PINNED_POOL_MB,
// default 1024) and handed out again to the next request of about their size.  Process-wide, thread-safe.
#pragma once
#include <cstddef>

void *pinned_block_alloc(size_t bytes);  // nullptr when cudaMallocHost fails
void pinned_block_free(void *p);         // nullptr is fine

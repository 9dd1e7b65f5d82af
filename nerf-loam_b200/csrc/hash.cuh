// Open-addressing hash sets of 64-bit keys with linear probing, shared by eval.cu (cell table of the nearest-neighbour search),
// overlap.cu (voxel sets of the keyframe overlap), ground.cu (column table of the vertical filter) and globalloc.cu (occupied
// voxels and lattice cells of the global localisation).  A slot holds NL_HASH_EMPTY until one atomicCAS claims it, and is never
// written again, so a plain load that sees a key sees it for good; a stale "empty" is resolved by the CAS.  The caller keeps the
// capacity a power of two and the load factor below 1 (every user here stays at or below 1/2), and never stores NL_HASH_EMPTY as a key.
#pragma once
#include <cstdint>

constexpr uint64_t NL_HASH_EMPTY = ~uint64_t(0);

__device__ __forceinline__ uint64_t nl_hash_mix(uint64_t z) {      // splitmix64 finaliser: the home slot of a key
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Adds k to the set; true when this call put it there (exactly one caller per distinct key sees true).
__device__ __forceinline__ bool nl_hash_insert(uint64_t *slots, uint64_t mask, uint64_t k) {
    for (uint64_t s = nl_hash_mix(k) & mask;; s = (s + 1) & mask) {
        const uint64_t h = slots[s];
        if (h == k) return false;
        if (h != NL_HASH_EMPTY) continue;
        const unsigned long long prev = atomicCAS((unsigned long long *)&slots[s], (unsigned long long)NL_HASH_EMPTY, (unsigned long long)k);
        if (prev == NL_HASH_EMPTY) return true;
        if (prev == k) return false;
    }
}

// Adds k to the set if absent and returns its slot, for callers that keep values beside the keys (ground.cu's column extents).
__device__ __forceinline__ uint64_t nl_hash_insert_slot(uint64_t *slots, uint64_t mask, uint64_t k) {
    for (uint64_t s = nl_hash_mix(k) & mask;; s = (s + 1) & mask) {
        const uint64_t h = slots[s];
        if (h == k) return s;
        if (h != NL_HASH_EMPTY) continue;
        const unsigned long long prev = atomicCAS((unsigned long long *)&slots[s], (unsigned long long)NL_HASH_EMPTY, (unsigned long long)k);
        if (prev == NL_HASH_EMPTY || prev == k) return s;
    }
}

// The slot of k, which must be in the set.
__device__ __forceinline__ uint64_t nl_hash_slot_of(const uint64_t *__restrict__ slots, uint64_t mask, uint64_t k) {
    uint64_t s = nl_hash_mix(k) & mask;
    while (slots[s] != k) s = (s + 1) & mask;
    return s;
}

__device__ __forceinline__ bool nl_hash_contains(const uint64_t *__restrict__ slots, uint64_t mask, uint64_t k) {
    for (uint64_t s = nl_hash_mix(k) & mask;; s = (s + 1) & mask) {
        const uint64_t h = slots[s];
        if (h == k) return true;
        if (h == NL_HASH_EMPTY) return false;
    }
}

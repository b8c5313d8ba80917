// Counter-based RNG shared by the device policy kernels and the host helper
// jss_host_masked_random().  One 32-bit draw per (seed, global env id, step index): the three
// counters are folded to 32 bits, combined with odd multipliers and passed through the
// murmur3 32-bit finaliser (~16 integer instructions on the GPU; a 64-bit splitmix variant cost
// ~40).  Stateless, so any env's action stream can be replayed on the host (the CPU oracle
// restates the same function for its replays).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define JSS_HD __host__ __device__
#else
#define JSS_HD
#endif

JSS_HD static inline uint32_t jss_fold32(uint64_t v) { return (uint32_t)v ^ ((uint32_t)(v >> 32) * 0x7FEB352Du); }

JSS_HD static inline uint32_t jss_hash3(uint64_t seed, uint64_t env, uint64_t ctr) {
    uint32_t h = jss_fold32(seed) ^ (jss_fold32(env) * 0x9E3779B1u + 0x85EBCA77u) ^ (jss_fold32(ctr) * 0xC2B2AE3Du + 0x27D4EB2Fu);
    h ^= h >> 16; h *= 0x85EBCA6Bu;
    h ^= h >> 13; h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h;
}

// The same hash with the launch-uniform part (seed, counter) folded once per launch on the host:
//   jss_hash3(seed, env, ctr) == jss_hash_env(jss_hash_key(seed, ctr), env)
JSS_HD static inline uint32_t jss_hash_key(uint64_t seed, uint64_t ctr) {
    return jss_fold32(seed) ^ (jss_fold32(ctr) * 0xC2B2AE3Du + 0x27D4EB2Fu);
}
JSS_HD static inline uint32_t jss_hash_env(uint32_t key, uint64_t env) {
    uint32_t h = key ^ (jss_fold32(env) * 0x9E3779B1u + 0x85EBCA77u);
    h ^= h >> 16; h *= 0x85EBCA6Bu;
    h ^= h >> 13; h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h;
}

// jss_hash_key with the seed already folded: jss_hash_key(seed, ctr) == jss_hash_key_folded(jss_fold32(seed), ctr), so a
// launch that varies the counter per env carries the seed in 32 bits
JSS_HD static inline uint32_t jss_hash_key_folded(uint32_t seed_folded, uint64_t ctr) {
    return seed_folded ^ (jss_fold32(ctr) * 0xC2B2AE3Du + 0x27D4EB2Fu);
}

// index in [0, count) -- multiply-high, no modulo bias worth speaking of
JSS_HD static inline uint32_t jss_pick(uint32_t h, uint32_t count) {
    return (uint32_t)(((uint64_t)h * (uint64_t)count) >> 32);
}

// the rules' exploration coin (dispatching.py:113): u = h / 2^32 < 0.1
#define JSS_COIN_THRESHOLD 429496730u

/* ransac_sample.h -- the RANSAC sample sets of the batched robust tracker, drawn on the device: the procedure of
 * util::create_random_array(8, 0, n - 1) (util/random_array.cc:46-88) over a counter-based generator.
 *
 * The reference seeds a fresh std::mt19937 from std::random_device on every draw, so its sample sets are not
 * reproducible; any seeded generator is as faithful, provided the draw procedure is the reference's.  Here the stream of
 * hypothesis `iter` of frame `b` under `seed` is SplitMix64 started from
 *     key = mix(mix(seed + G (b + 1)) + G (iter + 1)),   G = 0x9E3779B97F4A7C15, mix = SplitMix64's finaliser,
 * i.e. the j-th 64-bit draw (j = 1, 2, ...) is mix(key + j G), all arithmetic modulo 2^64.  Then:
 *   1. draw floor(8 * 1.2) = 9 unbiased integers in [0, n) (reject r < 2^64 mod n, take r mod n);
 *   2. sort them and drop duplicates; keep the 8 smallest when more than 8 remain;
 *   3. while fewer than 8 remain, draw until there are 9 values again and repeat step 2;
 *   4. Fisher-Yates shuffle: for i = 7 .. 1, swap v[i] with v[uniform(i + 1)], same stream.
 * The "8 smallest of 9" bias and the shuffle are the reference's.  n >= 8.  tests/robust_track_data.py restates it in
 * Python.  Plain integer arithmetic: nvcc, the host emulator and the restatement draw the same numbers.
 */
#ifndef PLP_RANSAC_SAMPLE_H
#define PLP_RANSAC_SAMPLE_H

#include <stdint.h>

#if defined(__CUDACC__)
#define RS_HD __host__ __device__ __forceinline__
#else
#define RS_HD static inline
#endif

#define RS_GOLDEN 0x9E3779B97F4A7C15ull

RS_HD uint64_t rs_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

/* the next 64-bit draw of the stream whose state is *s */
RS_HD uint64_t rs_next(uint64_t *s) {
    *s += RS_GOLDEN;
    return rs_mix(*s);
}

/* an unbiased integer in [0, n), n >= 1 */
RS_HD uint32_t rs_uniform(uint64_t *s, uint32_t n) {
    const uint64_t reject_below = (0ull - (uint64_t)n) % (uint64_t)n; /* 2^64 mod n */
    uint64_t r;
    do {
        r = rs_next(s);
    } while (r < reject_below);
    return (uint32_t)(r % (uint64_t)n);
}

RS_HD uint64_t rs_key(uint64_t seed, uint32_t b, uint32_t iter) {
    return rs_mix(rs_mix(seed + RS_GOLDEN * ((uint64_t)b + 1)) + RS_GOLDEN * ((uint64_t)iter + 1));
}

/* create_random_array(8, 0, n - 1) of hypothesis `iter` of frame `b`: 8 distinct indices in [0, n), shuffled */
RS_HD void rs_sample8(uint64_t seed, uint32_t b, uint32_t iter, uint32_t n, int32_t out[8]) {
    uint64_t s = rs_key(seed, b, iter);
    uint32_t v[9];
    int m = 0;
    while (m != 8) {
        while (m < 9) v[m++] = rs_uniform(&s, n);
        for (int i = 1; i < m; ++i) { /* insertion sort, then unique */
            const uint32_t x = v[i];
            int j = i - 1;
            while (j >= 0 && v[j] > x) {
                v[j + 1] = v[j];
                --j;
            }
            v[j + 1] = x;
        }
        int u = 1;
        for (int i = 1; i < m; ++i)
            if (v[i] != v[u - 1]) v[u++] = v[i];
        m = u > 8 ? 8 : u;
    }
    for (int i = 7; i >= 1; --i) {
        const uint32_t j = rs_uniform(&s, (uint32_t)i + 1);
        const uint32_t t = v[i];
        v[i] = v[j];
        v[j] = t;
    }
    for (int i = 0; i < 8; ++i) out[i] = (int32_t)v[i];
}

#endif

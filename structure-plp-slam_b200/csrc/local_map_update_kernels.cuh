// local_map_update_kernels.cuh -- device code of the batched local-map update (local_map_update.cu launches it):
// tracking_module::update_local_map (tracking_module.cc:837-906) and module::local_map_updater (local_map_updater.cc),
// monocular points, for the frames the local-map stage will start (local_map_kernels.cuh) from the same record:
//   the clean-up of erased tracked landmarks (:840-852) -> count_keyframe_weights (:89-108) ->
//   find_first_local_keyframes (:110-141) -> find_second_local_keyframes (:143-204) -> find_local_landmarks (:206-238)
// and the plp_track_local the local-map stage reads, with its last-frame and keyframe row mappings.
// Free of host-side CUDA runtime dependencies so that tests/cta_emu can compile the same text for the host.
//
// Kernels, in launch order:
//   lmu_vote_kernel    one CTA per frame: clears the frame's landmark table; votes in a shared open-addressing keyframe
//                      table; the first level in ascending keyframe index and the nearest keyframe; the second level in
//                      one warp; the row prefix of the local keyframes
//   lmu_dedup_kernel   grid (candidate chunks, frames): every candidate row's landmark into the frame's landmark table,
//                      keeping the smallest candidate position (atomicMin)
//   lmu_compact_kernel one CTA per frame: the first occurrences in candidate order (compact_in_order), the status, the
//                      frame's row count and keyframe local_idx block length
//   lmu_scan_kernel    one CTA: offsets and local_idx_offsets over the batch
//   lmu_fill_kernel    grid (row chunks, frames): the plp_track_local rows, local_lm, last_local_idx and local_idx
//
// Order: the reference walks the voted keyframes in the iteration order of an unordered_map keyed by pointer; here the
// first level is in ascending keyframe index (the caller fills the table in keyframe::id_ order), so ties for the
// nearest keyframe go to the lowest index.  Every other order is the reference's own.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "../../include/plpslam_b200.h"
#include "devmath.cuh"
#include "track_common.cuh"

namespace plp {

namespace lu {

constexpr int kThreads = 256;         // vote / compact / scan: one CTA
constexpr int kChunkThreads = 256;    // dedup / fill: one thread per candidate or row
constexpr int kMaxLocalKeyframes = 60;  // tracking_module.cc:873 max_num_local_keyfrms
constexpr int kMinReservedKeyframes = 64;  // a second level can bring the list to 63
constexpr int kEmpty = -1;

enum : int32_t { kStatusOk = 0, kStatusCapacity = 1, kStatusKeyframes = 2, kStatusNoVote = 3 };

struct UpdDev {
    int batch, cap, max_local, max_lkf;
    int vote_slots, lm_slots;          // powers of two: >= 2 x max_lkf, >= 2 x max_local
    // the tracking records of the batch (stage == nullptr: the record does not stand) and their rows' landmarks
    TrackRecord motion, kf, rb;
    const int32_t *n_kp;
    const int32_t *last_offsets;       // the motion call's plp_track_last offsets
    const int32_t *kf_of_frame, *kf_row_offsets;  // the keyframe call's table (null without a keyframe record)
    plp_track_map map;
    // scratch
    int32_t *cand_off;                 // batch x (max_lkf + 1): candidate position of each local keyframe's first row
    int32_t *hkey, *hpos, *hidx;       // batch x lm_slots: landmark, first candidate position, local index
    int32_t *uniq;                     // batch: distinct landmarks inserted
    int32_t *first_lm;                 // batch x max_local: the local list's landmarks, per frame
    int32_t *count, *lidx_len;         // batch: local rows, keyframe local_idx block length
    // outputs
    int32_t *nearest, *local_kf, *num_local_kf, *local_lm, *status;
    double *pos_w, *normal;
    float *min_d, *max_d, *max_raw;
    uint8_t *desc, *valid;
    int32_t *offsets, *last_local_idx, *local_idx, *local_idx_offsets;
};

// the frame runs update_local_map: the local-map stage would start it (same record, same gate)
__device__ __forceinline__ bool frame_active(const UpdDev &D, int b) {
    const TrackRecord &S = start_record(D, b);
    return S.num_valid[b] >= kNumMatchesThr && (!S.status || S.status[b] == 0);
}

__device__ __forceinline__ unsigned slot_of(int key, int slots) { return ((unsigned)key * 2654435761u) & (slots - 1); }

// the landmark held by keypoint i after the start record's discard_outliers, or -1
__device__ __forceinline__ int tracked_lm(const UpdDev &D, int b, int i) {
    const TrackRecord &S = start_record(D, b);
    const bool from_kf = ran(D.rb, b) || ran(D.kf, b);  // keyframe rows, else last-frame rows
    const int q = S.matched[(size_t)b * D.cap + i];
    if (q < 0) return -1;
    const int row = S.rows.offsets[row_block(S.rows, b)] + q;
    return from_kf ? D.map.kf_row_lm[row] : D.map.last_row_lm[row];
}

// the local index of landmark lm in frame b's table, or -1
__device__ __forceinline__ int lookup_local(const UpdDev &D, int b, int lm) {
    if (lm < 0) return -1;
    const size_t base = (size_t)b * D.lm_slots;
    unsigned h = slot_of(lm, D.lm_slots);
    for (int probe = 0; probe < D.lm_slots; ++probe) {
        const int k = D.hkey[base + h];
        if (k == lm) return D.hidx[base + h];
        if (k == kEmpty) return -1;
        h = (h + 1) & (D.lm_slots - 1);
    }
    return -1;
}

// the slot of landmark lm in frame b's table (it was inserted), or -1
__device__ __forceinline__ int find_slot(const UpdDev &D, int b, int lm) {
    const size_t base = (size_t)b * D.lm_slots;
    unsigned h = slot_of(lm, D.lm_slots);
    for (int probe = 0; probe < D.lm_slots; ++probe) {
        const int k = D.hkey[base + h];
        if (k == lm) return (int)h;
        if (k == kEmpty) return -1;
        h = (h + 1) & (D.lm_slots - 1);
    }
    return -1;
}

// Shared memory of lmu_vote_kernel: the vote table (keys, counts), the local keyframe list and its row counts.
__host__ __device__ inline size_t vote_smem_bytes(int vote_slots, int max_lkf) {
    return (size_t)vote_slots * 2 * sizeof(int32_t) + (size_t)max_lkf * 2 * sizeof(int32_t);
}

// Appends the first of cand[0, n) that is a keyframe, not erased and not in list[0, len) (add_second_local_keyframe,
// local_map_updater.cc:150-168); one warp, every lane calls it.  Returns the new length.
__device__ __forceinline__ int add_first_new(const UpdDev &D, const int32_t *cand, int n, int32_t *list, int len) {
    const int lane = threadIdx.x & 31;
    for (int c0 = 0; c0 < n; c0 += 32) {
        const int c = c0 + lane < n ? cand[c0 + lane] : -1;
        bool ok = c >= 0 && !D.map.kf_erased[c];
        for (int j = 0; ok && j < len; ++j) ok = list[j] != c;
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        if (bal) {
            const int first = __shfl_sync(0xffffffffu, c, __ffs(bal) - 1);
            if (lane == 0) list[len] = first;
            __syncwarp();
            return len + 1;
        }
    }
    return len;
}

__global__ void __launch_bounds__(kThreads, 1) lmu_vote_kernel(UpdDev D) {
    PLP_DYNAMIC_SMEM(smem_raw);
    int32_t *skey = reinterpret_cast<int32_t *>(smem_raw);
    int32_t *scnt = skey + D.vote_slots;
    int32_t *list = scnt + D.vote_slots;
    int32_t *nrows = list + D.max_lkf;
    __shared__ int s_voted, s_full, s_first, s_len;
    __shared__ unsigned long long s_best;
    const int b = blockIdx.x, tid = threadIdx.x;
    const bool active = frame_active(D, b);
    // the frame's landmark table starts empty
    const size_t hbase = (size_t)b * D.lm_slots;
    for (int s = tid; s < D.lm_slots; s += kThreads) {
        D.hkey[hbase + s] = kEmpty;
        D.hpos[hbase + s] = 0x7fffffff;
    }
    for (int s = tid; s < D.vote_slots; s += kThreads) {
        skey[s] = kEmpty;
        scnt[s] = 0;
    }
    if (tid == 0) {
        s_voted = s_full = s_first = 0;
        s_best = 0ull;
        D.uniq[b] = 0;
    }
    __syncthreads();
    // count_keyframe_weights over the tracked keypoints whose landmark survives the clean-up (tracking_module.cc:840-852)
    const int n = active ? D.n_kp[b] : 0;
    for (int i = tid; i < n; i += kThreads) {
        const int lm = tracked_lm(D, b, i);
        if (lm < 0 || D.map.lm_erased[lm]) continue;
        for (int o = D.map.obs_offsets[lm]; o < D.map.obs_offsets[lm + 1]; ++o) {
            const int kf = D.map.obs_kf[o];
            unsigned h = slot_of(kf, D.vote_slots);
            int probe = 0;
            for (; probe < D.vote_slots; ++probe) {
                const int k = atomicCAS(&skey[h], kEmpty, kf);
                if (k == kEmpty) atomicAdd(&s_voted, 1);
                if (k == kEmpty || k == kf) {
                    atomicAdd(&scnt[h], 1);
                    break;
                }
                h = (h + 1) & (D.vote_slots - 1);
            }
            if (probe == D.vote_slots) atomicOr(&s_full, 1);
        }
    }
    __syncthreads();
    const int status = !active ? kStatusOk
                       : s_voted == 0 ? kStatusNoVote
                       : (s_full || s_voted > D.max_lkf) ? kStatusKeyframes
                                                          : kStatusOk;
    const bool build = active && status == kStatusOk;
    // find_first_local_keyframes: the non-erased voted keyframes, ranked by index; nearest = largest weight, then lowest
    // index (the strict max_weight < weight over ascending indices)
    if (build) {
        for (int s = tid; s < D.vote_slots; s += kThreads)
            if (skey[s] != kEmpty && D.map.kf_erased[skey[s]]) scnt[s] = 0;  // erased: not a local keyframe
    }
    __syncthreads();
    if (build) {
        for (int s = tid; s < D.vote_slots; s += kThreads) {
            const int k = skey[s];
            if (k == kEmpty || scnt[s] == 0) continue;
            int rank = 0;
            for (int s2 = 0; s2 < D.vote_slots; ++s2) rank += (skey[s2] != kEmpty && scnt[s2] != 0 && skey[s2] < k);
            list[rank] = k;
            atomicAdd(&s_first, 1);
            atomicMax(&s_best, ((unsigned long long)(unsigned)scnt[s] << 32) | (unsigned)(0x7fffffff - k));
        }
    }
    __syncthreads();
    // find_second_local_keyframes (local_map_updater.cc:169-201) in warp 0; the cap is tested at the top of the loop
    if (tid < 32) {
        int len = s_first;
        if (build) {
            const int n_first = len;
            for (int j = 0; j < n_first; ++j) {
                if (kMaxLocalKeyframes < len) break;
                const int kf = list[j];
                const int c0 = D.map.cov_offsets[kf], h0 = D.map.child_offsets[kf];
                len = add_first_new(D, D.map.cov_kf + c0, D.map.cov_offsets[kf + 1] - c0, list, len);
                len = add_first_new(D, D.map.child_kf + h0, D.map.child_offsets[kf + 1] - h0, list, len);
                len = add_first_new(D, D.map.parent + kf, 1, list, len);  // -1 (no parent) is never added
            }
        }
        if (tid == 0) s_len = len;
    }
    __syncthreads();
    const int len = build ? s_len : 0;
    const size_t kbase = (size_t)b * D.max_lkf;
    for (int j = tid; j < len; j += kThreads) {
        const int kf = list[j];
        D.local_kf[kbase + j] = kf;
        nrows[j] = D.map.row_offsets[kf + 1] - D.map.row_offsets[kf];
    }
    __syncthreads();
    if (tid == 0) {
        // candidate position of each local keyframe's first row (find_local_landmarks walks them in list order)
        int32_t *co = D.cand_off + (size_t)b * (D.max_lkf + 1);
        int acc = 0;
        for (int j = 0; j < len; ++j) {
            co[j] = acc;
            acc += nrows[j];
        }
        co[len] = acc;
        D.num_local_kf[b] = len;
        D.nearest[b] = build && s_first > 0 ? 0x7fffffff - (int)(unsigned)(s_best & 0xffffffffu) : -1;
        D.status[b] = status;
    }
}

// find_local_landmarks (local_map_updater.cc:206-238): each candidate row's landmark, unless null or erased, goes into
// the frame's table with the smallest candidate position that holds it.  A table with more than max_local landmarks
// makes the frame's status 1 (lmu_compact_kernel); inserting stops there.
__global__ void __launch_bounds__(kChunkThreads) lmu_dedup_kernel(UpdDev D) {
    const int b = blockIdx.y;
    const int len = D.num_local_kf[b];
    const int32_t *co = D.cand_off + (size_t)b * (D.max_lkf + 1);
    const int total = co[len];
    const size_t hbase = (size_t)b * D.lm_slots;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < total; p += gridDim.x * blockDim.x) {
        if (__ldcg(&D.uniq[b]) > D.max_local) return;
        int lo = 0, hi = len - 1;  // the last local keyframe whose first candidate is <= p
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (co[mid] <= p) lo = mid; else hi = mid - 1;
        }
        const int kf = D.local_kf[(size_t)b * D.max_lkf + lo];
        const int lm = D.map.row_lm[D.map.row_offsets[kf] + (p - co[lo])];
        if (lm < 0 || D.map.lm_erased[lm]) continue;
        unsigned h = slot_of(lm, D.lm_slots);
        for (int probe = 0; probe < D.lm_slots; ++probe) {
            const int k = atomicCAS(&D.hkey[hbase + h], kEmpty, lm);
            if (k == kEmpty) atomicAdd(&D.uniq[b], 1);
            if (k == kEmpty || k == lm) {
                atomicMin(&D.hpos[hbase + h], p);
                break;
            }
            h = (h + 1) & (D.lm_slots - 1);
        }
    }
}

// The first occurrences in candidate order -> the frame's local list; the frame's status, row count and keyframe
// local_idx block length.
__global__ void __launch_bounds__(kThreads) lmu_compact_kernel(UpdDev D) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const int len = D.num_local_kf[b];
    const int32_t *co = D.cand_off + (size_t)b * (D.max_lkf + 1);
    const bool fits = D.uniq[b] <= D.max_local;
    const int total = fits ? co[len] : 0;
    const size_t hbase = (size_t)b * D.lm_slots, lbase = (size_t)b * D.max_local;
    int jk = 0, lm = -1, slot = -1;  // the local keyframe, landmark and slot of candidate p, found by take(p) for emit
    const int n_first = compact_in_order<kThreads>(
        total,
        [&](int p) {
            while (jk + 1 < len && co[jk + 1] <= p) ++jk;  // p ascends in every thread
            const int kf = D.local_kf[(size_t)b * D.max_lkf + jk];
            lm = D.map.row_lm[D.map.row_offsets[kf] + (p - co[jk])];
            if (lm < 0 || D.map.lm_erased[lm]) return false;
            slot = find_slot(D, b, lm);
            return slot >= 0 && D.hpos[hbase + slot] == p;
        },
        [&](int, int off) {
            D.first_lm[lbase + off] = lm;
            D.hidx[hbase + slot] = off;
        });
    if (tid == 0) {
        int status = D.status[b];
        if (status == kStatusOk && !fits) status = kStatusCapacity;
        D.status[b] = status;
        D.count[b] = status == kStatusOk ? n_first : 0;
        if (status != kStatusOk) {
            D.nearest[b] = -1;
            D.num_local_kf[b] = 0;
        }
        // a keyframe- or robust-started frame maps its keyframe's rows (the local-map stage reads that block)
        const bool kf_rows = ran(D.kf, b) && (!D.kf.status || D.kf.status[b] == 0);
        const int k = kf_rows ? D.kf_of_frame[b] : 0;
        D.lidx_len[b] = kf_rows ? D.kf_row_offsets[k + 1] - D.kf_row_offsets[k] : 0;
    }
}

// exclusive prefix of v over a block of kThreads threads (one round); total: the round's sum
template <int kThreadsT>
__device__ __forceinline__ int block_exclusive_scan(int v, int &total) {
    __shared__ int warp_tot[kThreadsT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    int before = 0;
    total = 0;
    for (int w = 0; w < kThreadsT / 32; ++w) {
        const int t = warp_tot[w];
        before += w < warp ? t : 0;
        total += t;
    }
    __syncthreads();
    return before + x - v;
}

__global__ void __launch_bounds__(kThreads) lmu_scan_kernel(UpdDev D) {
    int acc_rows = 0, acc_idx = 0;
    for (int b0 = 0; b0 < D.batch; b0 += kThreads) {
        const int b = b0 + threadIdx.x;
        int tot_rows, tot_idx;
        const int r = block_exclusive_scan<kThreads>(b < D.batch ? D.count[b] : 0, tot_rows);
        const int k = block_exclusive_scan<kThreads>(b < D.batch ? D.lidx_len[b] : 0, tot_idx);
        if (b < D.batch) {
            D.offsets[b] = acc_rows + r;
            D.local_idx_offsets[b] = acc_idx + k;
        }
        acc_rows += tot_rows;
        acc_idx += tot_idx;
    }
    if (threadIdx.x == 0) {
        D.offsets[D.batch] = acc_rows;
        D.local_idx_offsets[D.batch] = acc_idx;
    }
}

// The local rows from the landmark table, and the row mappings the local-map stage reads: last_local_idx for every
// plp_track_last row of the frame, local_idx for its keyframe's rows.
__global__ void __launch_bounds__(kChunkThreads) lmu_fill_kernel(UpdDev D) {
    const int b = blockIdx.y;
    const int stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = D.status[b] == kStatusOk;
    const int r0 = D.offsets[b], m = D.count[b];
    const size_t lbase = (size_t)b * D.max_local;
    for (int j = t0; j < m; j += stride) {
        const int lm = D.first_lm[lbase + j];
        const size_t r = (size_t)r0 + j;
        for (int c = 0; c < 3; ++c) {
            D.pos_w[3 * r + c] = D.map.pos_w[3 * (size_t)lm + c];
            D.normal[3 * r + c] = D.map.obs_mean_normal[3 * (size_t)lm + c];
        }
        D.min_d[r] = D.map.min_valid_dist[lm];
        D.max_d[r] = D.map.max_valid_dist[lm];
        D.max_raw[r] = D.map.max_valid_dist_raw[lm];
        const uint32_t *src = reinterpret_cast<const uint32_t *>(D.map.desc + 32 * (size_t)lm);
        uint32_t *dst = reinterpret_cast<uint32_t *>(D.desc + 32 * r);
        for (int w = 0; w < 8; ++w) dst[w] = src[w];
        D.valid[r] = 1;
        D.local_lm[r] = lm;
    }
    const int l0 = D.last_offsets[b], nl = D.last_offsets[b + 1] - l0;
    for (int j = t0; j < nl; j += stride)
        D.last_local_idx[l0 + j] = ok ? lookup_local(D, b, D.map.last_row_lm[l0 + j]) : -1;
    const int nk = D.lidx_len[b];
    if (nk > 0) {
        const int k0 = D.kf_row_offsets[D.kf_of_frame[b]], i0 = D.local_idx_offsets[b];
        for (int j = t0; j < nk; j += stride) D.local_idx[i0 + j] = ok ? lookup_local(D, b, D.map.kf_row_lm[k0 + j]) : -1;
    }
}

}  // namespace lu

}  // namespace plp

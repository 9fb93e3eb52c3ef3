// local_map_update_oracle.cc -- CPU restatement of tracking_module::update_local_map (tracking_module.cc:837-906) and
// module::local_map_updater (local_map_updater.cc:75-238) for one frame, monocular points, TEST INFRASTRUCTURE ONLY.
// Keyframes and landmarks are table indices; the voted keyframes are walked in ascending index, the canonical order that
// stands in for the reference's unordered_map<keyframe *, unsigned> iteration (DESIGN.md §3.17).
// tests/local_map_update_data.py calls it and holds an independent Python restatement it must equal.
#include <stdint.h>

#include <map>
#include <unordered_set>
#include <vector>

extern "C" {

// tracked_lm[n]: the landmark each keypoint holds after tracking (-1: none).  Returns 0 when no keyframe voted
// (acquire_local_map fails, :877-880), else 1 with out_kf[counts[0]] the local keyframes, out_lm[counts[1]] the local
// landmarks, counts[2] the nearest covisibility (-1: none) and counts[3] the number of voted keyframes.
int lmuo_update_local_map(int n, int K, int L, const int32_t *tracked_lm, const uint8_t *lm_erased,
                          const int32_t *obs_offsets, const int32_t *obs_kf, const uint8_t *kf_erased,
                          const int32_t *row_offsets, const int32_t *row_lm, const int32_t *cov_offsets,
                          const int32_t *cov_kf, const int32_t *child_offsets, const int32_t *child_kf,
                          const int32_t *parent, int32_t *out_kf, int32_t *out_lm, int32_t *counts) {
    (void)K;
    (void)L;
    // update_local_map's clean-up (:840-852): an erased landmark is dropped from the frame before the vote
    std::vector<int32_t> frm_lms(tracked_lm, tracked_lm + n);
    for (auto &lm : frm_lms)
        if (lm >= 0 && lm_erased[lm]) lm = -1;
    // count_keyframe_weights (local_map_updater.cc:89-108); std::map iterates in ascending keyframe index
    std::map<int32_t, unsigned> weights;
    for (int32_t lm : frm_lms) {
        if (lm < 0) continue;
        for (int32_t o = obs_offsets[lm]; o < obs_offsets[lm + 1]; ++o) ++weights[obs_kf[o]];
    }
    counts[0] = counts[1] = 0;
    counts[2] = -1;
    counts[3] = (int32_t)weights.size();
    if (weights.empty()) return 0;
    // find_first_local_keyframes (:110-141)
    std::vector<int32_t> first;
    std::unordered_set<int32_t> marked;  // keyframe::local_map_update_identifier == frm_id_
    unsigned max_weight = 0;
    int32_t nearest = -1;
    for (const auto &kw : weights) {
        if (kf_erased[kw.first]) continue;
        first.push_back(kw.first);
        marked.insert(kw.first);
        if (max_weight < kw.second) {
            max_weight = kw.second;
            nearest = kw.first;
        }
    }
    // find_second_local_keyframes (:143-204)
    std::vector<int32_t> second;
    auto add = [&](int32_t kf) {
        if (kf < 0 || kf_erased[kf] || marked.count(kf)) return false;
        marked.insert(kf);
        second.push_back(kf);
        return true;
    };
    const unsigned max_num_local_keyfrms = 60;  // tracking_module.cc:873
    for (int32_t kf : first) {
        if (max_num_local_keyfrms < first.size() + second.size()) break;
        for (int32_t c = cov_offsets[kf]; c < cov_offsets[kf + 1]; ++c)
            if (add(cov_kf[c])) break;
        for (int32_t c = child_offsets[kf]; c < child_offsets[kf + 1]; ++c)
            if (add(child_kf[c])) break;
        add(parent[kf]);
    }
    std::vector<int32_t> local_kf = first;
    local_kf.insert(local_kf.end(), second.begin(), second.end());
    // find_local_landmarks (:206-238)
    std::unordered_set<int32_t> seen;  // landmark::identifier_in_local_map_update_ == frm_id_
    int32_t m = 0;
    for (int32_t kf : local_kf)
        for (int32_t r = row_offsets[kf]; r < row_offsets[kf + 1]; ++r) {
            const int32_t lm = row_lm[r];
            if (lm < 0 || lm_erased[lm] || !seen.insert(lm).second) continue;
            out_lm[m++] = lm;
        }
    for (size_t j = 0; j < local_kf.size(); ++j) out_kf[j] = local_kf[j];
    counts[0] = (int32_t)local_kf.size();
    counts[1] = m;
    counts[2] = nearest;
    return 1;
}

// The host path a batched loop without the device update runs after its motion call: for each of B frames, its tracked
// landmarks (matched[b * cap + i], a row of the frame's last-frame block, for i < n_kp[b]), update_local_map when the
// motion track succeeded (num_valid >= 20), and the last_local_idx of the frame's rows.  A frame that did not succeed,
// whose keyframes got no vote or whose list exceeds max_local gets an empty list.  out_offsets: B + 1; out_lm:
// B x max_local; out_last_local_idx: one per last-frame row.
void lmuo_update_batch(int B, int cap, int K, int L, int max_local, const int32_t *n_kp, const int32_t *matched,
                       const int32_t *num_valid, const int32_t *last_offsets, const int32_t *last_row_lm,
                       const uint8_t *lm_erased, const int32_t *obs_offsets, const int32_t *obs_kf,
                       const uint8_t *kf_erased, const int32_t *row_offsets, const int32_t *row_lm,
                       const int32_t *cov_offsets, const int32_t *cov_kf, const int32_t *child_offsets,
                       const int32_t *child_kf, const int32_t *parent, int32_t *out_offsets, int32_t *out_lm,
                       int32_t *out_last_local_idx) {
    std::vector<int32_t> tracked(cap), kf_buf(K > 0 ? K : 1), lm_buf(L > 0 ? L : 1), pos(L > 0 ? L : 1, -1);
    int32_t counts[4];
    out_offsets[0] = 0;
    for (int b = 0; b < B; ++b) {
        const int32_t l0 = last_offsets[b], l1 = last_offsets[b + 1];
        int32_t m = 0;
        if (num_valid[b] >= 20) {
            for (int i = 0; i < n_kp[b]; ++i) {
                const int32_t q = matched[(size_t)b * cap + i];
                tracked[i] = q >= 0 ? last_row_lm[l0 + q] : -1;
            }
            if (lmuo_update_local_map(n_kp[b], K, L, tracked.data(), lm_erased, obs_offsets, obs_kf, kf_erased,
                                      row_offsets, row_lm, cov_offsets, cov_kf, child_offsets, child_kf, parent,
                                      kf_buf.data(), lm_buf.data(), counts) &&
                counts[1] <= max_local)
                m = counts[1];
        }
        for (int32_t j = 0; j < m; ++j) {
            out_lm[(size_t)b * max_local + j] = lm_buf[j];
            pos[lm_buf[j]] = j;
        }
        for (int32_t r = l0; r < l1; ++r) out_last_local_idx[r] = last_row_lm[r] >= 0 ? pos[last_row_lm[r]] : -1;
        for (int32_t j = 0; j < m; ++j) pos[lm_buf[j]] = -1;
        out_offsets[b + 1] = out_offsets[b] + m;
    }
}

}  // extern "C"

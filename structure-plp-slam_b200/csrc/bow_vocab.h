// bow_vocab.h -- internal: the device-resident DBoW2 vocabulary, shared by bow.cu (transform, bow_tree) and
// keyframe_track.cu (frame::compute_bow of the frames the batched keyframe tracker runs on).
#pragma once
#include "common.cuh"
#include "bow_kernels.cuh"

struct plp_bow_vocab {
    plp_ctx *ctx = nullptr;
    int k = 0, L = 0, num_nodes = 0, num_words = 0, max_children = 0;
    uint8_t *d_desc = nullptr;          // num_nodes x 32
    uint32_t *d_child_begin = nullptr;  // num_nodes + 1
    uint32_t *d_children = nullptr;     // num_nodes - 1 node ids, grouped by parent, ascending id inside a group
    float *d_weight = nullptr;          // num_nodes
    int32_t *d_word_id = nullptr;       // num_nodes (-1 for inner nodes)
};

namespace plp {

inline VocabDev vocab_dev(const plp_bow_vocab *v) {
    VocabDev V;
    V.desc = v->d_desc;
    V.child_begin = v->d_child_begin;
    V.children = v->d_children;
    V.weight = v->d_weight;
    V.word_id = v->d_word_id;
    return V;
}

// lanes per descriptor in the transform: the smallest power of two >= the widest node (at least 4, at most a warp)
inline int transform_group(const plp_bow_vocab *v) {
    return v->max_children <= 4 ? 4 : v->max_children <= 8 ? 8 : v->max_children <= 16 ? 16 : 32;
}

}  // namespace plp

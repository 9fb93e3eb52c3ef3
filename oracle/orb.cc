// oracle/orb.cc -- CPU restatement of feature::orb_extractor (TEST INFRASTRUCTURE ONLY).
//
// Follows /root/reference/src/PLPSLAM/feature/orb_extractor.cc, orb_extractor_node.cc,
// orb_params.cc:86-128, util/trigonometric.h.  The OpenCV primitives the reference calls
// (cv::resize INTER_LINEAR, cv::FAST 9_16 + NMS, cv::GaussianBlur 7x7 sigma 2, cv::fastAtan2) are
// third-party code absent from /root/reference; they are restated from OpenCV's published
// fixed-point algorithms and pinned bit-exactly against cv2 4.13 in tests/test_orb_oracle.py.
#include "orb.h"

#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <list>
#include <vector>

#define PLP_BRIEF_TABLE static const signed char
#include "brief_pattern.inc"

namespace {

inline int cvFloor(double v) {
    int i = (int)v;
    return i - (i > v);
}
inline int cvCeil(double v) {
    int i = (int)v;
    return i + (i < v);
}
inline int cvRoundF(float v) { return (int)std::lrintf(v); }
inline int cvRoundD(double v) { return (int)std::lrint(v); }

struct Image {
    std::vector<uint8_t> data;
    int w = 0, h = 0;
    const uint8_t *row(int y) const { return data.data() + (size_t)y * w; }
    uint8_t *row(int y) { return data.data() + (size_t)y * w; }
    uint8_t at(int y, int x) const { return data[(size_t)y * w + x]; }
};

// ---------------------------------------------------------------- cv::resize INTER_LINEAR 8UC1
void resize_linear(const uint8_t *src, int sw, int sh, int sstep, uint8_t *dst, int dw, int dh, int dstep) {
    const double inv_scale_x = (double)dw / sw, inv_scale_y = (double)dh / sh;
    const double scale_x = 1. / inv_scale_x, scale_y = 1. / inv_scale_y;
    std::vector<int> xofs(dw), yofs(dh);
    std::vector<short> ialpha(2 * dw), ibeta(2 * dh);
    for (int dx = 0; dx < dw; ++dx) {
        float fx = (float)((dx + 0.5) * scale_x - 0.5);
        int sx = cvFloor(fx);
        fx -= sx;
        if (sx < 0) {
            fx = 0;
            sx = 0;
        }
        if (sx >= sw - 1) {
            fx = 0;
            sx = sw - 1;
        }
        xofs[dx] = sx;
        ialpha[2 * dx] = (short)cvRoundF((1.f - fx) * 2048);
        ialpha[2 * dx + 1] = (short)cvRoundF(fx * 2048);
    }
    for (int dy = 0; dy < dh; ++dy) {
        float fy = (float)((dy + 0.5) * scale_y - 0.5);
        int sy = cvFloor(fy);
        fy -= sy;
        // OpenCV clamps the row index when fetching rows (clip), the weights stay as computed
        yofs[dy] = sy;
        ibeta[2 * dy] = (short)cvRoundF((1.f - fy) * 2048);
        ibeta[2 * dy + 1] = (short)cvRoundF(fy * 2048);
    }
    std::vector<int> r0(dw), r1(dw);
    for (int dy = 0; dy < dh; ++dy) {
        const int sy0 = std::min(std::max(yofs[dy], 0), sh - 1);
        const int sy1 = std::min(std::max(yofs[dy] + 1, 0), sh - 1);
        const uint8_t *S0 = src + (size_t)sy0 * sstep, *S1 = src + (size_t)sy1 * sstep;
        for (int dx = 0; dx < dw; ++dx) {
            const int sx = xofs[dx];
            const int sx1 = std::min(sx + 1, sw - 1);
            const int a0 = ialpha[2 * dx], a1 = ialpha[2 * dx + 1];
            r0[dx] = S0[sx] * a0 + S0[sx1] * a1;
            r1[dx] = S1[sx] * a0 + S1[sx1] * a1;
        }
        const int b0 = ibeta[2 * dy], b1 = ibeta[2 * dy + 1];
        uint8_t *D = dst + (size_t)dy * dstep;
        for (int dx = 0; dx < dw; ++dx)
            D[dx] = (uint8_t)((((b0 * (r0[dx] >> 4)) >> 16) + ((b1 * (r1[dx] >> 4)) >> 16) + 2) >> 2);
    }
}

// ---------------------------------------------------------------- cv::FAST TYPE_9_16
const int kRingDx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
const int kRingDy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};

// m = max over the 16 contiguous 9-arcs of min(arc differences), both polarities
inline int fast_arc_max_min(const uint8_t *p, int step) {
    int d[32];
    const int v = p[0];
    for (int k = 0; k < 16; ++k) d[k] = d[k + 16] = v - p[kRingDy[k] * step + kRingDx[k]];
    int best = -255;
    for (int k = 0; k < 16; ++k) {
        int mn = 255, mx = -255;
        for (int i = 0; i < 9; ++i) {
            mn = std::min(mn, d[k + i]);
            mx = std::max(mx, d[k + i]);
        }
        best = std::max(best, std::max(mn, -mx));
    }
    return best;
}

// m-map of the tested interior of an ROI (-1 for the untested 3-px margin)
void fast_m_map(const uint8_t *img, int w, int h, int step, std::vector<int16_t> &mm) {
    mm.assign((size_t)w * h, -1);
    for (int y = 3; y < h - 3; ++y)
        for (int x = 3; x < w - 3; ++x) mm[(size_t)y * w + x] = (int16_t)fast_arc_max_min(img + (size_t)y * step + x, step);
}

// cv::FAST(roi, kps, thr, nonmax): corner iff m > thr, score = m - 1 (0 for non-corners / margin),
// NMS keeps a corner iff its score is strictly greater than all 8 neighbours'; row-major output.
int fast_detect_from_map(const std::vector<int16_t> &mm, int w, int h, int thr, bool nonmax,
                         std::vector<orc_keypoint> &out) {
    auto score = [&](int y, int x) {
        const int m = mm[(size_t)y * w + x];
        return m > thr ? m - 1 : 0;
    };
    int cnt = 0;
    for (int y = 3; y < h - 3; ++y)
        for (int x = 3; x < w - 3; ++x) {
            if (!(mm[(size_t)y * w + x] > thr)) continue;
            const int sc = score(y, x);
            if (nonmax) {
                bool keep = true;
                for (int dy = -1; dy <= 1 && keep; ++dy)
                    for (int dx = -1; dx <= 1; ++dx) {
                        if (!dx && !dy) continue;
                        if (!(sc > score(y + dy, x + dx))) {
                            keep = false;
                            break;
                        }
                    }
                if (!keep) continue;
            }
            orc_keypoint kp;
            kp.x = (float)x;
            kp.y = (float)y;
            kp.size = 7.f;
            kp.angle = -1.f;
            kp.response = nonmax ? (float)sc : 0.f;  // cv::FAST only scores corners when NMS is on
            kp.octave = 0;
            kp.class_id = -1;
            out.push_back(kp);
            ++cnt;
        }
    return cnt;
}

int fast_detect(const uint8_t *img, int w, int h, int step, int thr, bool nonmax, std::vector<orc_keypoint> &out) {
    if (w < 7 || h < 7) return 0;
    std::vector<int16_t> mm;
    fast_m_map(img, w, h, step, mm);
    return fast_detect_from_map(mm, w, h, thr, nonmax, out);
}

// ---------------------------------------------------------------- cv::GaussianBlur fixed point
inline int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) {
        if (p < 0) p = -p;
        if (p >= len) p = 2 * (len - 1) - p;
    }
    return p;
}

void gaussian_blur_q8(const uint8_t *src, int w, int h, int sstep, uint8_t *dst, int dstep, const int *k, int ksize) {
    const int r = ksize / 2;
    std::vector<uint32_t> tmp((size_t)w * h);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint32_t acc = 0;
            for (int i = -r; i <= r; ++i) acc += (uint32_t)src[(size_t)y * sstep + reflect101(x + i, w)] * k[i + r];
            tmp[(size_t)y * w + x] = acc;  // Q8, <= 255*256
        }
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint32_t acc = 0;
            for (int i = -r; i <= r; ++i) acc += tmp[(size_t)reflect101(y + i, h) * w + x] * k[i + r];
            dst[(size_t)y * dstep + x] = (uint8_t)((acc + 32768u) >> 16);
        }
}

const int kGauss7[7] = {18, 34, 48, 56, 48, 34, 18};   // 7x7, sigma 2 (orb_extractor.cc:149)
const int kGauss5[5] = {14, 62, 104, 62, 14};          // 5x5, sigma 1 (binary_descriptor_custom.cpp:355)

// ---------------------------------------------------------------- cv::fastAtan2 (degrees)
float fast_atan2(float y, float x) {
    const float scale = (float)(180.0 / 3.14159265358979323846);
    const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale,
                p5 = 0.1555786518463281f * scale, p7 = -0.04432655554792128f * scale;
    const float ax = std::abs(x), ay = std::abs(y);
    float a, c, c2;
    if (ax >= ay) {
        c = ay / (ax + (float)DBL_EPSILON);
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = ax / (ay + (float)DBL_EPSILON);
        c2 = c * c;
        a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

// ---------------------------------------------------------------- util/trigonometric.h:36-78
constexpr float _PI = 3.14159265358979f;
constexpr float _PI_2 = _PI / 2.0f;
constexpr float _TWO_PI = 2.0f * _PI;
constexpr float _INV_TWO_PI = 1.0f / _TWO_PI;
constexpr float _THREE_PI_2 = 3.0f * _PI_2;

inline float poly_cos(float v) {
    constexpr float c1 = 0.99940307f, c2 = -0.49558072f, c3 = 0.03679168f;
    const float v2 = v * v;
    return c1 + v2 * (c2 + c3 * v2);
}
float util_cos(float v) {
    v = v - cvFloor(v * _INV_TWO_PI) * _TWO_PI;
    v = (0.0f < v) ? v : -v;
    if (v < _PI_2) return poly_cos(v);
    if (v < _PI) return -poly_cos(_PI - v);
    if (v < _THREE_PI_2) return -poly_cos(v - _PI);
    return poly_cos(_TWO_PI - v);
}
float util_sin(float v) { return util_cos(_PI_2 - v); }

// ---------------------------------------------------------------- orb_extractor
constexpr int kFastPatchSize = 31;       // orb_extractor.h:156
constexpr int kFastHalfPatch = 15;       // :158
constexpr int kOrbPatchRadius = 19;      // :161

struct Node {  // orb_extractor_node.h
    std::vector<orc_keypoint> keypts;
    int bx = 0, by = 0, ex = 0, ey = 0;
    std::list<Node>::iterator iter;
    bool is_leaf = false;
    long creation = 0;  // oracle tie-break (replaces the node address in std::sort, orb_extractor.cc:529)
};

struct Extractor {
    orc_orb_params p;
    std::vector<float> scale_factors, inv_scale_factors, level_sigma_sq, inv_level_sigma_sq;
    std::vector<unsigned> num_keypts_per_level;
    std::vector<int> u_max;
    long creation_counter = 0;

    explicit Extractor(const orc_orb_params &pp) : p(pp) {
        const unsigned L = p.num_levels;
        scale_factors.assign(L, 1.0f);
        inv_scale_factors.assign(L, 1.0f);
        level_sigma_sq.assign(L, 1.0f);
        inv_level_sigma_sq.assign(L, 1.0f);
        // orb_params.cc:86-128
        for (unsigned l = 1; l < L; ++l) scale_factors[l] = p.scale_factor * scale_factors[l - 1];
        for (unsigned l = 1; l < L; ++l) inv_scale_factors[l] = (1.0f / p.scale_factor) * inv_scale_factors[l - 1];
        float s = 1.0f;
        for (unsigned l = 1; l < L; ++l) {
            s = p.scale_factor * s;
            level_sigma_sq[l] = s * s;
            inv_level_sigma_sq[l] = 1.0f / (s * s);
        }
        // orb_extractor.cc:244-253
        num_keypts_per_level.resize(L);
        double desired = p.max_num_keypts * (1.0 - 1.0 / p.scale_factor) /
                         (1.0 - std::pow(1.0 / p.scale_factor, static_cast<double>(L)));
        unsigned total = 0;
        for (unsigned l = 0; l + 1 < L; ++l) {
            num_keypts_per_level[l] = (unsigned)std::round(desired);
            total += num_keypts_per_level[l];
            desired *= 1.0 / p.scale_factor;
        }
        num_keypts_per_level[L - 1] = (unsigned)std::max((int)p.max_num_keypts - (int)total, 0);
        // orb_extractor.cc:270-286
        u_max.resize(kFastHalfPatch + 1);
        const unsigned vmax = (unsigned)std::floor(kFastHalfPatch * std::sqrt(2.0) / 2 + 1);
        const unsigned vmin = (unsigned)std::ceil(kFastHalfPatch * std::sqrt(2.0) / 2);
        for (unsigned v = 0; v <= vmax; ++v)
            u_max[v] = (int)std::round(std::sqrt((double)kFastHalfPatch * kFastHalfPatch - (double)v * v));
        for (unsigned v = kFastHalfPatch, v0 = 0; vmin <= v; --v) {
            while (u_max[v0] == u_max[v0 + 1]) ++v0;
            u_max[v] = v0;
            ++v0;
        }
    }

    // orb_extractor.cc:315-326
    std::vector<Image> pyramid(const uint8_t *img, int rows, int cols, int step) const {
        std::vector<Image> pyr(p.num_levels);
        pyr[0].w = cols;
        pyr[0].h = rows;
        pyr[0].data.resize((size_t)rows * cols);
        for (int y = 0; y < rows; ++y) std::memcpy(pyr[0].row(y), img + (size_t)y * step, cols);
        for (unsigned l = 1; l < p.num_levels; ++l) {
            const double scale = scale_factors[l];
            const int w = (int)std::round(cols * 1.0 / scale), h = (int)std::round(rows * 1.0 / scale);
            pyr[l].w = w;
            pyr[l].h = h;
            pyr[l].data.resize((size_t)w * h);
            resize_linear(pyr[l - 1].data.data(), pyr[l - 1].w, pyr[l - 1].h, pyr[l - 1].w, pyr[l].data.data(), w, h, w);
        }
        return pyr;
    }

    // orb_extractor_node.cc:31-80
    static std::array<Node, 4> divide(const Node &n) {
        const unsigned half_x = (unsigned)cvCeil((n.ex - n.bx) / 2.0);
        const unsigned half_y = (unsigned)cvCeil((n.ey - n.by) / 2.0);
        std::array<Node, 4> c;
        c[0].bx = n.bx; c[0].by = n.by; c[0].ex = n.bx + half_x; c[0].ey = n.by + half_y;
        c[1].bx = n.bx + half_x; c[1].by = n.by; c[1].ex = n.ex; c[1].ey = n.by + half_y;
        c[2].bx = n.bx; c[2].by = n.by + half_y; c[2].ex = n.bx + half_x; c[2].ey = n.ey;
        c[3].bx = n.bx + half_x; c[3].by = n.by + half_y; c[3].ex = n.ex; c[3].ey = n.ey;
        for (const auto &k : n.keypts) {
            unsigned idx = 0;
            if (n.bx + half_x <= k.x) idx += 1;
            if (n.by + half_y <= k.y) idx += 2;
            c[idx].keypts.push_back(k);
        }
        return c;
    }

    // orb_extractor.cc:639-657
    void assign_children(std::array<Node, 4> &children, std::list<Node> &nodes,
                         std::vector<std::pair<int, Node *>> &leaf_pool) {
        for (auto &c : children) {
            if (c.keypts.empty()) continue;
            c.creation = creation_counter++;
            nodes.push_front(c);
            if (c.keypts.size() == 1) continue;
            leaf_pool.emplace_back((int)c.keypts.size(), &nodes.front());
            nodes.front().iter = nodes.begin();
        }
    }

    // orb_extractor.cc:468-555 (+ initialize_nodes :557-637, find_keypoints_with_max_response :659-685)
    std::vector<orc_keypoint> distribute(const std::vector<orc_keypoint> &cands, int min_x, int max_x, int min_y,
                                         int max_y, unsigned num_keypts) {
        creation_counter = 0;
        std::list<Node> nodes;
        {
            const double ratio = static_cast<double>(max_x - min_x) / (max_y - min_y);
            double delta_x, delta_y;
            unsigned num_x_grid, num_y_grid;
            if (ratio > 1) {
                num_x_grid = (unsigned)std::round(ratio);
                num_y_grid = 1;
                delta_x = static_cast<double>(max_x - min_x) / num_x_grid;
                delta_y = max_y - min_y;
            } else {
                num_x_grid = 1;
                num_y_grid = (unsigned)std::round(1 / ratio);
                delta_x = max_x - min_y;  // sic (orb_extractor.cc:580)
                delta_y = static_cast<double>(max_y - min_y) / num_y_grid;
            }
            const unsigned num_initial = num_x_grid * num_y_grid;
            std::vector<Node *> initial(num_initial);
            for (unsigned i = 0; i < num_initial; ++i) {
                Node node;
                const unsigned ix = i % num_x_grid, iy = i / num_x_grid;
                node.bx = (int)(delta_x * ix);
                node.by = (int)(delta_y * iy);
                node.ex = (int)(delta_x * (ix + 1));
                node.ey = (int)(delta_y * (iy + 1));
                node.creation = creation_counter++;
                nodes.push_back(node);
                initial[i] = &nodes.back();
            }
            for (const auto &k : cands) {
                const unsigned ix = (unsigned)(k.x / delta_x), iy = (unsigned)(k.y / delta_y);
                initial.at(ix + iy * num_x_grid)->keypts.push_back(k);
            }
            for (auto it = nodes.begin(); it != nodes.end();) {
                if (it->keypts.empty()) {
                    it = nodes.erase(it);
                    continue;
                }
                it->is_leaf = (it->keypts.size() == 1);
                ++it;
            }
        }
        std::vector<std::pair<int, Node *>> leaf_pool;
        bool is_filled = false;
        while (true) {
            const unsigned prev_size = (unsigned)nodes.size();
            auto iter = nodes.begin();
            leaf_pool.clear();
            while (iter != nodes.end()) {
                if (iter->is_leaf) {
                    ++iter;
                    continue;
                }
                auto children = divide(*iter);
                assign_children(children, nodes, leaf_pool);
                iter = nodes.erase(iter);
            }
            if (num_keypts <= nodes.size() || nodes.size() == prev_size) {
                is_filled = true;
                break;
            }
            if (num_keypts < nodes.size() + leaf_pool.size()) {
                is_filled = false;
                break;
            }
        }
        while (!is_filled) {
            const unsigned prev_size = (unsigned)nodes.size();
            auto prev_pool = leaf_pool;
            leaf_pool.clear();
            // std::sort(rbegin, rend) on (count, node*): descending count; ties on the node address are
            // replaced by the oracle rule "later-created node first".
            std::stable_sort(prev_pool.begin(), prev_pool.end(),
                             [](const std::pair<int, Node *> &a, const std::pair<int, Node *> &b) {
                                 if (a.first != b.first) return a.first > b.first;
                                 return a.second->creation > b.second->creation;
                             });
            for (const auto &pl : prev_pool) {
                auto children = divide(*pl.second);
                assign_children(children, nodes, leaf_pool);
                nodes.erase(pl.second->iter);
                if (num_keypts <= nodes.size()) {
                    is_filled = true;
                    break;
                }
            }
            if (is_filled || num_keypts <= nodes.size() || nodes.size() == prev_size) {
                is_filled = true;
                break;
            }
        }
        std::vector<orc_keypoint> result;
        result.reserve(nodes.size());
        for (auto &node : nodes) {
            orc_keypoint best = node.keypts.at(0);
            double max_response = best.response;
            for (size_t k = 1; k < node.keypts.size(); ++k)
                if (node.keypts[k].response > max_response) {
                    best = node.keypts[k];
                    max_response = node.keypts[k].response;
                }
            result.push_back(best);
        }
        return result;
    }

    // orb_extractor.cc:708-735
    float ic_angle(const Image &im, float px, float py) const {
        int m_01 = 0, m_10 = 0;
        const int cx = cvRoundF(px), cy = cvRoundF(py);
        const uint8_t *center = im.row(cy) + cx;
        for (int u = -kFastHalfPatch; u <= kFastHalfPatch; ++u) m_10 += u * center[u];
        const int step = im.w;
        for (int v = 1; v <= kFastHalfPatch; ++v) {
            int v_sum = 0;
            const int d = u_max[v];
            for (int u = -d; u <= d; ++u) {
                const int val_plus = center[u + v * step], val_minus = center[u - v * step];
                v_sum += (val_plus - val_minus);
                m_10 += u * (val_plus + val_minus);
            }
            m_01 += v * v_sum;
        }
        return fast_atan2((float)m_01, (float)m_10);
    }

    // orb_extractor.cc:747-807
    void describe(const Image &blurred, const orc_keypoint &kp, uint8_t *desc) const {
        const float angle = (float)(kp.angle * M_PI / 180.0);
        const float cos_angle = util_cos(angle), sin_angle = util_sin(angle);
        const uint8_t *center = blurred.row(cvRoundF(kp.y)) + cvRoundF(kp.x);
        const int step = blurred.w;
        auto value = [&](int x, int y) {
            const int r = cvRoundF((float)x * sin_angle + (float)y * cos_angle);
            const int c = cvRoundF((float)x * cos_angle - (float)y * sin_angle);
            return center[r * step + c];
        };
        for (int i = 0; i < 32; ++i) {
            int val = 0;
            for (int b = 0; b < 8; ++b) {
                const int k = i * 8 + b;
                val |= (value(kBriefX1[k], kBriefY1[k]) < value(kBriefX2[k], kBriefY2[k])) << b;
            }
            desc[i] = (uint8_t)val;
        }
    }

    // orb_extractor.cc:328-466 for one level: FAST over 64-px cells with 6-px overlap
    std::vector<orc_keypoint> fast_candidates(const Image &im, unsigned level, const uint8_t *mask, int mask_step) const {
        constexpr unsigned overlap = 6, cell_size = 64;
        const float scale_factor = scale_factors[level];
        auto is_in_mask = [&](unsigned y, unsigned x) {
            return mask[(size_t)(int)(y * scale_factor) * mask_step + (int)(x * scale_factor)] == 0;
        };
        const unsigned min_border_x = kOrbPatchRadius, min_border_y = kOrbPatchRadius;
        const unsigned max_border_x = im.w - kOrbPatchRadius, max_border_y = im.h - kOrbPatchRadius;
        const unsigned width = max_border_x - min_border_x, height = max_border_y - min_border_y;
        const unsigned num_cols = (unsigned)std::ceil(width / cell_size) + 1;
        const unsigned num_rows = (unsigned)std::ceil(height / cell_size) + 1;
        std::vector<orc_keypoint> out;
        for (unsigned i = 0; i < num_rows; ++i) {
            const unsigned min_y = min_border_y + i * cell_size;
            if (max_border_y - overlap <= min_y) continue;
            unsigned max_y = min_y + cell_size + overlap;
            if (max_border_y < max_y) max_y = max_border_y;
            for (unsigned j = 0; j < num_cols; ++j) {
                const unsigned min_x = min_border_x + j * cell_size;
                if (max_border_x - overlap <= min_x) continue;
                unsigned max_x = min_x + cell_size + overlap;
                if (max_border_x < max_x) max_x = max_border_x;
                if (mask) {
                    if (is_in_mask(min_y, min_x) || is_in_mask(max_y, min_x) || is_in_mask(min_y, max_x) ||
                        is_in_mask(max_y, max_x))
                        continue;
                }
                std::vector<orc_keypoint> in_cell;
                const uint8_t *roi = im.row(min_y) + min_x;
                const int cw = (int)(max_x - min_x), ch = (int)(max_y - min_y);
                if (cw >= 7 && ch >= 7) {
                    std::vector<int16_t> mm;
                    fast_m_map(roi, cw, ch, im.w, mm);
                    fast_detect_from_map(mm, cw, ch, (int)p.ini_fast_thr, true, in_cell);
                    if (in_cell.empty()) fast_detect_from_map(mm, cw, ch, (int)p.min_fast_thr, true, in_cell);
                }
                if (in_cell.empty()) continue;
                for (auto &k : in_cell) {
                    k.x += j * cell_size;
                    k.y += i * cell_size;
                    if (mask && is_in_mask((unsigned)(min_border_y + k.y), (unsigned)(min_border_x + k.x))) continue;
                    out.push_back(k);
                }
            }
        }
        return out;
    }
};

}  // namespace

extern "C" {

void orc_resize_linear(const uint8_t *src, int sw, int sh, int sstep, uint8_t *dst, int dw, int dh, int dstep) {
    resize_linear(src, sw, sh, sstep, dst, dw, dh, dstep);
}

int orc_fast9_16(const uint8_t *img, int w, int h, int step, int thr, int nonmax, orc_keypoint *out, int cap) {
    std::vector<orc_keypoint> v;
    fast_detect(img, w, h, step, thr, nonmax != 0, v);
    const int n = std::min((int)v.size(), cap);
    std::copy(v.begin(), v.begin() + n, out);
    return (int)v.size();
}

void orc_gaussian_blur_7x7(const uint8_t *src, int w, int h, int sstep, uint8_t *dst, int dstep) {
    gaussian_blur_q8(src, w, h, sstep, dst, dstep, kGauss7, 7);
}
void orc_gaussian_blur_5x5(const uint8_t *src, int w, int h, int sstep, uint8_t *dst, int dstep) {
    gaussian_blur_q8(src, w, h, sstep, dst, dstep, kGauss5, 5);
}

float orc_fast_atan2(float y, float x) { return fast_atan2(y, x); }
float orc_util_cos(float v) { return util_cos(v); }
float orc_util_sin(float v) { return util_sin(v); }

void orc_orb_tables(const orc_orb_params *p, float *scale_factors, float *inv_scale_factors, float *level_sigma_sq,
                    float *inv_level_sigma_sq, uint32_t *num_keypts_per_level, int32_t *u_max16) {
    Extractor e(*p);
    for (unsigned l = 0; l < p->num_levels; ++l) {
        if (scale_factors) scale_factors[l] = e.scale_factors[l];
        if (inv_scale_factors) inv_scale_factors[l] = e.inv_scale_factors[l];
        if (level_sigma_sq) level_sigma_sq[l] = e.level_sigma_sq[l];
        if (inv_level_sigma_sq) inv_level_sigma_sq[l] = e.inv_level_sigma_sq[l];
        if (num_keypts_per_level) num_keypts_per_level[l] = e.num_keypts_per_level[l];
    }
    if (u_max16)
        for (int v = 0; v <= 15; ++v) u_max16[v] = e.u_max[v];
}

void orc_orb_level_sizes(const orc_orb_params *p, int rows, int cols, int32_t *w_out, int32_t *h_out) {
    Extractor e(*p);
    for (unsigned l = 0; l < p->num_levels; ++l) {
        if (l == 0) {
            w_out[l] = cols;
            h_out[l] = rows;
        } else {
            const double scale = e.scale_factors[l];
            w_out[l] = (int)std::round(cols * 1.0 / scale);
            h_out[l] = (int)std::round(rows * 1.0 / scale);
        }
    }
}

int orc_orb_distribute(const orc_orb_params *p, const orc_keypoint *cands, int n, int min_x, int max_x, int min_y,
                       int max_y, unsigned num_keypts, orc_keypoint *out) {
    Extractor e(*p);
    std::vector<orc_keypoint> c(cands, cands + n);
    const auto r = e.distribute(c, min_x, max_x, min_y, max_y, num_keypts);
    std::copy(r.begin(), r.end(), out);
    return (int)r.size();
}

float orc_orb_ic_angle(const orc_orb_params *p, const uint8_t *img, int w, int h, float px, float py) {
    Extractor e(*p);
    Image im;
    im.w = w;
    im.h = h;
    im.data.assign(img, img + (size_t)w * h);
    return e.ic_angle(im, px, py);
}

void orc_orb_describe(const orc_orb_params *p, const uint8_t *blurred, int w, int h, const orc_keypoint *kp,
                      uint8_t *desc) {
    Extractor e(*p);
    Image im;
    im.w = w;
    im.h = h;
    im.data.assign(blurred, blurred + (size_t)w * h);
    e.describe(im, *kp, desc);
}

int orc_orb_extract(const orc_orb_params *p, const uint8_t *img, int rows, int cols, int step, const uint8_t *mask,
                    int mask_step, orc_keypoint *kps_out, uint8_t *desc_out, int cap, uint8_t *pyramid_out,
                    orc_keypoint *cands_out, int cands_cap, int32_t *cands_per_level, int32_t *kps_per_level) {
    // orb_extractor.cc:73-160
    if (!img || rows <= 0 || cols <= 0) return 0;
    Extractor e(*p);
    const auto pyr = e.pyramid(img, rows, cols, step);
    if (pyramid_out) {
        size_t off = 0;
        for (const auto &im : pyr) {
            std::memcpy(pyramid_out + off, im.data.data(), im.data.size());
            off += im.data.size();
        }
    }
    std::vector<std::vector<orc_keypoint>> all(p->num_levels);
    int cand_total = 0;
    for (unsigned level = 0; level < p->num_levels; ++level) {
        const Image &im = pyr[level];
        if (im.w <= 2 * kOrbPatchRadius || im.h <= 2 * kOrbPatchRadius) {
            if (cands_per_level) cands_per_level[level] = 0;
            continue;
        }
        const auto cands = e.fast_candidates(im, level, mask, mask_step);
        if (cands_per_level) cands_per_level[level] = (int)cands.size();
        if (cands_out)
            for (const auto &c : cands)
                if (cand_total < cands_cap) cands_out[cand_total++] = c;
        const int min_bx = kOrbPatchRadius, min_by = kOrbPatchRadius;
        const int max_bx = im.w - kOrbPatchRadius, max_by = im.h - kOrbPatchRadius;
        std::vector<orc_keypoint> kl;
        if (!cands.empty()) kl = e.distribute(cands, min_bx, max_bx, min_by, max_by, e.num_keypts_per_level[level]);
        const unsigned scaled_patch_size = (unsigned)(kFastPatchSize * e.scale_factors[level]);
        for (auto &k : kl) {
            k.x += min_bx;
            k.y += min_by;
            k.octave = (int)level;
            k.size = (float)scaled_patch_size;
        }
        all[level] = kl;
    }
    for (unsigned level = 0; level < p->num_levels; ++level)
        for (auto &k : all[level]) k.angle = e.ic_angle(pyr[level], k.x, k.y);
    int n = 0;
    for (unsigned level = 0; level < p->num_levels; ++level) {
        if (kps_per_level) kps_per_level[level] = (int)all[level].size();
        if (all[level].empty()) continue;
        Image blurred;
        blurred.w = pyr[level].w;
        blurred.h = pyr[level].h;
        blurred.data.resize(pyr[level].data.size());
        gaussian_blur_q8(pyr[level].data.data(), blurred.w, blurred.h, blurred.w, blurred.data.data(), blurred.w, kGauss7, 7);
        for (auto &k : all[level]) {
            if (n >= cap) return -1;
            e.describe(blurred, k, desc_out + 32 * (size_t)n);
            if (level != 0) {  // orb_extractor.cc:695-706
                const float s = e.scale_factors[level];
                k.x *= s;
                k.y *= s;
            }
            kps_out[n++] = k;
        }
    }
    return n;
}

}  // extern "C"

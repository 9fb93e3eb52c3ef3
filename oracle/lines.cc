// oracle/lines.cc -- CPU restatement of the LSD + LBD line front end (TEST INFRASTRUCTURE ONLY, see oracle.h).
//
// Reference (paths under /root/reference/src/PLPSLAM):
//   feature/line_extractor.cc:88-160                       LineFeatureTracker::extract_LSD_LBD
//   feature/line_descriptor/LSDDetector_custom.cpp:76-102  checkLineExtremes
//   feature/line_descriptor/LSDDetector_custom.cpp:225-320 LSDDetectorC::detectImpl (with LSDOptions)
//   feature/line_descriptor/binary_descriptor_custom.cpp:217-258 (weights), 347-408 (pyramid, Sobel, binaryConversion),
//                                                        518-679 (computeImpl), 1018-1364 (computeLBD)
// Third party, absent from /root/reference: cv::LineSegmentDetector (OpenCV imgproc/src/lsd.cpp).  Restated from the
// published algorithm (Grompone von Gioi, Jakubowicz, Morel, Randall: "LSD: a Line Segment Detector", IPOL 2012) in
// the form OpenCV ships it (refine = LSD_REFINE_STD: density refinement, no NFA pass) and pinned against
// cv2 4.13 createLineSegmentDetector(1, 0.5, 0.6, 2.0, 22.5, 1.0, 0.6, 1024) in tests/test_lines_oracle.py.
//
// Two evaluation modes (orc_lsd_config):
//   "cv" mode  {seed_order 1, libm 1, sum_order 0}: what cv2 4.13 + glibc do on this machine -> used ONLY to pin this
//              restatement against cv2 (std::sort seed order, libm cosf/sinf, sequential sums, swap-remove compaction).
//   "det" mode {0, 0, 1}: the portable determinism rules the CUDA path implements bit-exactly: seeds ordered by gradient
//              bin (descending) with raster order inside a bin (the bin lists of the original LSD and of OpenCV 3.4,
//              the version the reference's README names), trigonometry by the library's detmath.h, sums accumulated in 32
//              strided partials and combined by a fixed xor-tree, order-preserving compaction.
#include "lines.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "detmath.h"
#include "orb.h"

namespace {

constexpr double kPi = 3.14159265358979323846;
constexpr double kNotDef = -1024.0;
constexpr double k3_2Pi = 4.71238898038;   // M_3_2_PI as lsd.cpp spells it
constexpr double k2Pi = 6.28318530718;     // M_2__PI as lsd.cpp spells it
constexpr double kDegToRads = 0.017453292519943295769236907684;

inline int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) {
        if (p < 0) p = -p;
        if (p >= len) p = 2 * (len - 1) - p;
    }
    return p;
}

// cv::GaussianBlur on CV_8U: Q8 separable fixed point, exact horizontal pass, vertical pass rounded (V + 2^15) >> 16
void blur_q8(const uint8_t *src, int w, int h, int sstep, uint8_t *dst, int dstep, const int *k, int ksize) {
    const int r = ksize / 2;
    std::vector<uint32_t> tmp((size_t)w * h);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint32_t acc = 0;
            for (int i = -r; i <= r; ++i) acc += (uint32_t)src[(size_t)y * sstep + reflect101(x + i, w)] * k[i + r];
            tmp[(size_t)y * w + x] = acc;
        }
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint32_t acc = 0;
            for (int i = -r; i <= r; ++i) acc += tmp[(size_t)reflect101(y + i, h) * w + x] * k[i + r];
            dst[(size_t)y * dstep + x] = (uint8_t)((acc + 32768u) >> 16);
        }
}

// sigma = 0.6 / 0.5 = 1.2, ksize = 1 + 2*ceil(1.2*sqrt(6 ln 10)) = 11; Q8 taps measured from cv2 (sum 256)
const int kGauss11[11] = {0, 0, 4, 21, 60, 86, 60, 21, 4, 0, 0};
const int kGauss5[5] = {14, 62, 104, 62, 14};

struct Cfg {
    bool std_sort, libm, lane_sums;
};

struct RegPt {
    int x, y;
    double angle, modgrad;
};

struct Rect {
    double x1, y1, x2, y2, width, x, y, theta, dx, dy, prec, p;
};

struct NormPoint {
    int x, y, norm;
};

// sum_{i<n} f(i): sequentially (cv) or as 32 strided partial sums combined by an xor-butterfly (what a warp does)
template <class F>
double ordered_sum(size_t n, bool lanes, F f) {
    if (!lanes) {
        double s = 0;
        for (size_t i = 0; i < n; ++i) s += f(i);
        return s;
    }
    double p[32];
    for (int l = 0; l < 32; ++l) p[l] = 0;
    for (size_t i = 0; i < n; ++i) p[i & 31] += f(i);
    for (int off = 16; off >= 1; off >>= 1)
        for (int l = 0; l < off; ++l) p[l] = p[l] + p[l + off];
    return p[0];
}

struct Lsd {
    int w = 0, h = 0;
    Cfg cfg{};
    std::vector<double> angles, modgrad;
    std::vector<uint8_t> used;
    std::vector<NormPoint> ordered;

    double cosd(double a) const { return cfg.libm ? std::cos(a) : det_cos(a); }
    double sind(double a) const { return cfg.libm ? std::sin(a) : det_sin(a); }
    // lsd.cpp: `sumdx += cos(float(angle))` resolves to the float overload
    float cosf_(float a) const { return cfg.libm ? cosf(a) : (float)det_cos((double)a); }
    float sinf_(float a) const { return cfg.libm ? sinf(a) : (float)det_sin((double)a); }

    void ll_angle(const uint8_t *img, double threshold, unsigned n_bins, int32_t *bins_out) {
        angles.assign((size_t)w * h, kNotDef);
        modgrad.assign((size_t)w * h, 0.0);
        double max_grad = -1;
        for (int y = 0; y < h - 1; ++y)
            for (int x = 0; x < w - 1; ++x) {
                const int DA = img[(size_t)(y + 1) * w + x + 1] - img[(size_t)y * w + x];
                const int BC = img[(size_t)y * w + x + 1] - img[(size_t)(y + 1) * w + x];
                const int gx = DA + BC, gy = DA - BC;
                const double norm = std::sqrt((gx * gx + gy * gy) / 4.0);
                modgrad[(size_t)y * w + x] = norm;
                if (norm <= threshold) {
                    angles[(size_t)y * w + x] = kNotDef;
                } else {
                    angles[(size_t)y * w + x] = (double)orc_fast_atan2((float)gx, (float)-gy) * kDegToRads;
                    if (norm > max_grad) max_grad = norm;
                }
            }
        const double bin_coef = (max_grad > 0) ? double(n_bins - 1) / max_grad : 0;
        ordered.clear();
        ordered.reserve((size_t)(w - 1) * (h - 1));
        for (int y = 0; y < h - 1; ++y)
            for (int x = 0; x < w - 1; ++x) {
                const int i = int(modgrad[(size_t)y * w + x] * bin_coef);
                ordered.push_back({x, y, i});
                if (bins_out) bins_out[(size_t)y * w + x] = i;
            }
        if (cfg.std_sort)
            std::sort(ordered.begin(), ordered.end(), [](const NormPoint &a, const NormPoint &b) { return a.norm > b.norm; });
        else
            std::stable_sort(ordered.begin(), ordered.end(),
                             [](const NormPoint &a, const NormPoint &b) { return a.norm > b.norm; });
    }

    bool is_aligned(int x, int y, double theta, double prec) const {
        if (x < 0 || y < 0 || x >= w || y >= h) return false;
        const double a = angles[(size_t)y * w + x];
        if (a == kNotDef) return false;
        double n_theta = theta - a;
        if (n_theta < 0) n_theta = -n_theta;
        if (n_theta > k3_2Pi) {
            n_theta -= k2Pi;
            if (n_theta < 0) n_theta = -n_theta;
        }
        return n_theta <= prec;
    }

    // debug trace (orc_debug_lsd_trace): bounding box / count of every pixel accepted while one seed is processed
    bool tracing = false;
    int tb[4] = {0, 0, 0, 0};
    long taccepted = 0;
    void trace_px(int x, int y) {
        if (!tracing) return;
        tb[0] = std::min(tb[0], x);
        tb[1] = std::min(tb[1], y);
        tb[2] = std::max(tb[2], x);
        tb[3] = std::max(tb[3], y);
        ++taccepted;
    }

    void region_grow(int sx, int sy, std::vector<RegPt> &reg, double &reg_angle, double prec) {
        reg.clear();
        trace_px(sx, sy);
        reg_angle = angles[(size_t)sy * w + sx];
        reg.push_back({sx, sy, reg_angle, modgrad[(size_t)sy * w + sx]});
        float sumdx = float(cosd(reg_angle));
        float sumdy = float(sind(reg_angle));
        used[(size_t)sy * w + sx] = 1;
        for (size_t i = 0; i < reg.size(); ++i) {
            const int px = reg[i].x, py = reg[i].y;
            const int xx_min = std::max(px - 1, 0), xx_max = std::min(px + 1, w - 1);
            const int yy_min = std::max(py - 1, 0), yy_max = std::min(py + 1, h - 1);
            for (int yy = yy_min; yy <= yy_max; ++yy)
                for (int xx = xx_min; xx <= xx_max; ++xx) {
                    uint8_t &u = used[(size_t)yy * w + xx];
                    if (u != 1 && is_aligned(xx, yy, reg_angle, prec)) {
                        const double angle = angles[(size_t)yy * w + xx];
                        u = 1;
                        trace_px(xx, yy);
                        reg.push_back({xx, yy, angle, modgrad[(size_t)yy * w + xx]});
                        sumdx += cosf_(float(angle));
                        sumdy += sinf_(float(angle));
                        reg_angle = (double)orc_fast_atan2(sumdy, sumdx) * kDegToRads;
                    }
                }
        }
    }

    static double angle_diff_signed(double a, double b) {
        double diff = a - b;
        while (diff <= -kPi) diff += k2Pi;
        while (diff > kPi) diff -= k2Pi;
        return diff;
    }
    static double dist(double x1, double y1, double x2, double y2) {
        return std::sqrt((x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1));
    }
    static double dist_sq(double x1, double y1, double x2, double y2) {
        return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1);
    }

    double get_theta(const std::vector<RegPt> &reg, double x, double y, double reg_angle, double prec) const {
        const bool L = cfg.lane_sums;
        const double Ixx = ordered_sum(reg.size(), L, [&](size_t i) {
            const double dy = double(reg[i].y) - y;
            return dy * dy * reg[i].modgrad;
        });
        const double Iyy = ordered_sum(reg.size(), L, [&](size_t i) {
            const double dx = double(reg[i].x) - x;
            return dx * dx * reg[i].modgrad;
        });
        // lsd.cpp accumulates Ixy -= dx*dy*w: the negated sum of the same products (negation is exact)
        const double Ixy = -ordered_sum(reg.size(), L, [&](size_t i) {
            const double dx = double(reg[i].x) - x, dy = double(reg[i].y) - y;
            return dx * dy * reg[i].modgrad;
        });
        const double lambda = 0.5 * (Ixx + Iyy - std::sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
        double theta = (std::fabs(Ixx) > std::fabs(Iyy)) ? double(orc_fast_atan2(float(lambda - Ixx), float(Ixy)))
                                                         : double(orc_fast_atan2(float(Ixy), float(lambda - Iyy)));
        theta *= kDegToRads;
        if (std::fabs(angle_diff_signed(theta, reg_angle)) > prec) theta += kPi;
        return theta;
    }

    void region2rect(const std::vector<RegPt> &reg, double reg_angle, double prec, double p, Rect &rec) const {
        const bool L = cfg.lane_sums;
        double x = ordered_sum(reg.size(), L, [&](size_t i) { return double(reg[i].x) * reg[i].modgrad; });
        double y = ordered_sum(reg.size(), L, [&](size_t i) { return double(reg[i].y) * reg[i].modgrad; });
        const double sum = ordered_sum(reg.size(), L, [&](size_t i) { return reg[i].modgrad; });
        x /= sum;
        y /= sum;
        const double theta = get_theta(reg, x, y, reg_angle, prec);
        const double dx = cosd(theta), dy = sind(theta);
        double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
        for (size_t i = 0; i < reg.size(); ++i) {
            const double regdx = double(reg[i].x) - x, regdy = double(reg[i].y) - y;
            const double l = regdx * dx + regdy * dy;
            const double wv = -regdx * dy + regdy * dx;
            if (l > l_max) l_max = l;
            else if (l < l_min) l_min = l;
            if (wv > w_max) w_max = wv;
            else if (wv < w_min) w_min = wv;
        }
        rec.x1 = x + l_min * dx;
        rec.y1 = y + l_min * dy;
        rec.x2 = x + l_max * dx;
        rec.y2 = y + l_max * dy;
        rec.width = w_max - w_min;
        rec.x = x;
        rec.y = y;
        rec.theta = theta;
        rec.dx = dx;
        rec.dy = dy;
        rec.prec = prec;
        rec.p = p;
        if (rec.width < 1.0) rec.width = 1.0;
    }

    bool reduce_region_radius(std::vector<RegPt> &reg, double reg_angle, double prec, double p, Rect &rec, double density,
                              double density_th) {
        const double xc = double(reg[0].x), yc = double(reg[0].y);
        const double r1 = dist_sq(xc, yc, rec.x1, rec.y1), r2 = dist_sq(xc, yc, rec.x2, rec.y2);
        double rad_sq = r1 > r2 ? r1 : r2;
        while (density < density_th) {
            rad_sq *= 0.75 * 0.75;
            if (cfg.lane_sums) {  // order-preserving compaction (a ballot/prefix compaction on the GPU)
                size_t o = 0;
                for (size_t i = 0; i < reg.size(); ++i) {
                    if (dist_sq(xc, yc, double(reg[i].x), double(reg[i].y)) > rad_sq)
                        used[(size_t)reg[i].y * w + reg[i].x] = 0;
                    else
                        reg[o++] = reg[i];
                }
                reg.resize(o);
            } else {  // lsd.cpp: swap with the last element, pop, re-test the swapped-in element
                for (size_t i = 0; i < reg.size(); ++i) {
                    if (dist_sq(xc, yc, double(reg[i].x), double(reg[i].y)) > rad_sq) {
                        used[(size_t)reg[i].y * w + reg[i].x] = 0;
                        std::swap(reg[i], reg[reg.size() - 1]);
                        reg.pop_back();
                        --i;
                    }
                }
            }
            if (reg.size() < 2) return false;
            region2rect(reg, reg_angle, prec, p, rec);
            density = double(reg.size()) / (dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
        }
        return true;
    }

    bool refine(std::vector<RegPt> &reg, double reg_angle, double prec, double p, Rect &rec, double density_th) {
        double density = double(reg.size()) / (dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
        if (density >= density_th) return true;
        const double xc = double(reg[0].x), yc = double(reg[0].y);
        const double ang_c = reg[0].angle;
        const bool L = cfg.lane_sums;
        int n = 0;
        for (size_t i = 0; i < reg.size(); ++i) {
            used[(size_t)reg[i].y * w + reg[i].x] = 0;
            if (dist(xc, yc, reg[i].x, reg[i].y) < rec.width) ++n;
        }
        const double sum = ordered_sum(reg.size(), L, [&](size_t i) {
            return dist(xc, yc, reg[i].x, reg[i].y) < rec.width ? angle_diff_signed(reg[i].angle, ang_c) : 0.0;
        });
        const double s_sum = ordered_sum(reg.size(), L, [&](size_t i) {
            if (!(dist(xc, yc, reg[i].x, reg[i].y) < rec.width)) return 0.0;
            const double d = angle_diff_signed(reg[i].angle, ang_c);
            return d * d;
        });
        const double mean_angle = sum / double(n);
        const double tau = 2.0 * std::sqrt((s_sum - 2.0 * mean_angle * sum) / double(n) + mean_angle * mean_angle);
        const int sx = reg[0].x, sy = reg[0].y;
        region_grow(sx, sy, reg, reg_angle, tau);
        if (reg.size() < 2) return false;
        region2rect(reg, reg_angle, prec, p, rec);
        density = double(reg.size()) / (dist(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
        if (density < density_th) return reduce_region_radius(reg, reg_angle, prec, p, rec, density, density_th);
        return true;
    }
};

constexpr double kScale = 0.5, kSigmaScale = 0.6, kQuant = 2.0, kAngTh = 22.5, kDensityTh = 0.6;
constexpr unsigned kBins = 1024;

void scaled_image(const uint8_t *img, int w, int h, int step, std::vector<uint8_t> &out, int &sw, int &sh) {
    std::vector<uint8_t> g((size_t)w * h);
    blur_q8(img, w, h, step, g.data(), w, kGauss11, 11);
    // resize(..., Size(), 0.5, 0.5, INTER_LINEAR_EXACT): dsize = round(w * 0.5), ties to even, so a dimension n = 3 (mod 4)
    // gets a last destination row / column with one source row / column (n = 1 (mod 4) drops the last source one).
    // At exactly 1/2 cv2 resizes by area over the source pixels that exist (derived from cv2 4.13 with impulses,
    // exhaustive value pairs in the last row and column and the corner, see test_lines_oracle.py):
    //   full 2x2 block:                          (s + 2) >> 2            (fixed point, ties up)
    //   last row or column, 2 source pixels:     s / 2, ties to even     (float sum / count, cvRound)
    //   corner, 1 source pixel:                  the pixel
    sw = (int)std::lrint(w * kScale);
    sh = (int)std::lrint(h * kScale);
    out.assign((size_t)sw * sh, 0);
    for (int y = 0; y < sh; ++y)
        for (int x = 0; x < sw; ++x) {
            const int x0 = 2 * x, x1 = std::min(2 * x + 1, w - 1);
            const int y0 = 2 * y, y1 = std::min(2 * y + 1, h - 1);
            int s = g[(size_t)y0 * w + x0];
            if (x1 != x0) s += g[(size_t)y0 * w + x1];
            if (y1 != y0) s += g[(size_t)y1 * w + x0];
            if (x1 != x0 && y1 != y0) s += g[(size_t)y1 * w + x1];
            const int n = (x1 != x0 ? 2 : 1) * (y1 != y0 ? 2 : 1);
            out[(size_t)y * sw + x] = (uint8_t)(n == 4 ? (s + 2) >> 2 : n == 2 ? (s + ((s >> 1) & 1)) >> 1 : s);
        }
}

int lsd_detect(const uint8_t *img, int w, int h, int step, const orc_lsd_config *c, std::vector<float> &segs,
               std::vector<int32_t> *trace = nullptr) {
    Lsd L;
    L.tracing = trace != nullptr;
    L.cfg = {c->seed_order != 0, c->libm_float != 0, c->sum_order != 0};
    std::vector<uint8_t> scaled;
    scaled_image(img, w, h, step, scaled, L.w, L.h);
    const double prec = kPi * kAngTh / 180;
    const double p = kAngTh / 180;
    const double rho = kQuant / std::sin(prec);
    L.ll_angle(scaled.data(), rho, kBins, nullptr);
    const double log_nt = 5 * (std::log10(double(L.w)) + std::log10(double(L.h))) / 2 + std::log10(11.0);
    const size_t min_reg_size = size_t(-log_nt / std::log10(p));
    L.used.assign((size_t)L.w * L.h, 0);
    std::vector<RegPt> reg;
    int32_t pos = -1;
    for (const NormPoint &pt : L.ordered) {
        ++pos;
        const size_t a = (size_t)pt.y * L.w + pt.x;
        if (L.used[a] != 0 || L.angles[a] == kNotDef) continue;
        double reg_angle;
        if (trace) {
            L.tb[0] = L.tb[1] = 1 << 30;
            L.tb[2] = L.tb[3] = -1;
            L.taccepted = 0;
        }
        // one record per processed seed: position in the order list, x, y, first region size, pixels accepted in total
        // (all growths), final region size (marks left), bounding box of everything accepted, segment emitted
        auto rec_out = [&](size_t first_n, size_t final_n, int emitted) {
            if (!trace) return;
            const int32_t r[11] = {pos, pt.x, pt.y, (int32_t)first_n, (int32_t)L.taccepted, (int32_t)final_n,
                                   L.tb[0], L.tb[1], L.tb[2], L.tb[3], emitted};
            trace->insert(trace->end(), r, r + 11);
        };
        L.region_grow(pt.x, pt.y, reg, reg_angle, prec);
        const size_t first_n = reg.size();
        if (reg.size() < min_reg_size) {
            rec_out(first_n, reg.size(), 0);
            continue;
        }
        Rect rec;
        L.region2rect(reg, reg_angle, prec, p, rec);
        if (!L.refine(reg, reg_angle, prec, p, rec, kDensityTh)) {
            rec_out(first_n, reg.size(), 0);
            continue;
        }
        rec_out(first_n, reg.size(), 1);
        rec.x1 += 0.5;
        rec.y1 += 0.5;
        rec.x2 += 0.5;
        rec.y2 += 0.5;
        rec.x1 /= kScale;
        rec.y1 /= kScale;
        rec.x2 /= kScale;
        rec.y2 /= kScale;
        segs.push_back(float(rec.x1));
        segs.push_back(float(rec.y1));
        segs.push_back(float(rec.x2));
        segs.push_back(float(rec.y2));
    }
    return (int)(segs.size() / 4);
}

// LSDDetector_custom.cpp:76-102
void check_line_extremes(float *e, int width, int height) {
    if (e[0] < 0) e[0] = 0;
    if (e[0] >= width) e[0] = (float)width - 1.0f;
    if (e[2] < 0) e[2] = 0;
    if (e[2] >= width) e[2] = (float)width - 1.0f;
    if (e[1] < 0) e[1] = 0;
    if (e[1] >= height) e[1] = (float)height - 1.0f;
    if (e[3] < 0) e[3] = 0;
    if (e[3] >= height) e[3] = (float)height - 1.0f;
}

// LSDDetector_custom.cpp:266-300 for octave 0 (octaveScale = pow(2.f, 0) = 1)
int make_keylines(const std::vector<float> &segs, int w, int h, const orc_lsd_config *c, double min_length,
                  std::vector<orc_keyline> &out) {
    int class_counter = -1;
    for (size_t k = 0; k < segs.size() / 4; ++k) {
        float e[4] = {segs[4 * k], segs[4 * k + 1], segs[4 * k + 2], segs[4 * k + 3]};
        check_line_extremes(e, w, h);
        const double ddx = (double)(e[0] - e[2]), ddy = (double)(e[1] - e[3]);
        const double length = (double)(float)std::sqrt(ddx * ddx + ddy * ddy);
        if (!(length > min_length)) continue;
        orc_keyline kl;
        kl.start_x = e[0];
        kl.start_y = e[1];
        kl.end_x = e[2];
        kl.end_y = e[3];
        kl.s_oct_x = e[0];
        kl.s_oct_y = e[1];
        kl.e_oct_x = e[2];
        kl.e_oct_y = e[3];
        kl.line_length = (float)length;
        // cv::LineIterator (8-connected) between the cvRound-ed end points, both inside the image: max(|dx|,|dy|) + 1
        const int x0 = (int)std::lrintf(e[0]), y0 = (int)std::lrintf(e[1]);
        const int x1 = (int)std::lrintf(e[2]), y1 = (int)std::lrintf(e[3]);
        kl.num_pixels = std::max(std::abs(x1 - x0), std::abs(y1 - y0)) + 1;
        const float ay = kl.end_y - kl.start_y, ax = kl.end_x - kl.start_x;
        kl.angle = c->libm_float ? (float)std::atan2((double)ay, (double)ax) : (float)det_atan2((double)ay, (double)ax);
        kl.class_id = ++class_counter;
        kl.octave = 0;
        kl.size = (kl.end_x - kl.start_x) * (kl.end_y - kl.start_y);
        kl.response = kl.line_length / (float)std::max(w, h);
        kl.pt_x = (kl.end_x + kl.start_x) / 2;
        kl.pt_y = (kl.end_y + kl.start_y) / 2;
        out.push_back(kl);
    }
    return (int)out.size();
}

// ------------------------------------------------------------------------------------------------ LBD
const int kCombinations[32][2] = {{0, 1}, {0, 2}, {0, 3}, {0, 4}, {0, 5}, {0, 6}, {1, 2}, {1, 3}, {1, 4}, {1, 5}, {1, 6},
                                  {2, 3}, {2, 4}, {2, 5}, {2, 6}, {2, 7}, {2, 8}, {3, 4}, {3, 5}, {3, 6}, {3, 7}, {3, 8},
                                  {4, 5}, {4, 6}, {4, 7}, {4, 8}, {5, 6}, {5, 7}, {5, 8}, {6, 7}, {6, 8}, {7, 8}};
constexpr int kBands = 9, kBandWidth = 7;

void lbd_weights(float *gauss_l /*21*/, float *gauss_g /*63*/) {
    // binary_descriptor_custom.cpp:229-257; note the integer divisions: u = (21-1)/2 = 10, sigma = (15)/2 = 7; u = 31 = sigma
    double u = (kBandWidth * 3 - 1) / 2;
    double sigma = (kBandWidth * 2 + 1) / 2;
    double inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < kBandWidth * 3; ++i) {
        const double dis = i - u;
        gauss_l[i] = (float)std::exp(dis * dis * inv);  // stored as double in the reference, always read through (float)
    }
    u = (kBands * kBandWidth - 1) / 2;
    sigma = u;
    inv = -1 / (2 * sigma * sigma);
    for (int i = 0; i < kBands * kBandWidth; ++i) {
        const double dis = i - u;
        gauss_g[i] = (float)std::exp(dis * dis * inv);
    }
}

void lbd_one(const int16_t *dximg, const int16_t *dyimg, int w, int h, const orc_keyline &kl, bool libm, const float *gl,
             const float *gg, float *des /*72*/) {
    const short height_lsp = kBandWidth * kBands;
    float band[8][kBands];
    std::memset(band, 0, sizeof(band));
    const short image_w = (short)(w - 1), image_h = (short)(h - 1);
    const short length_lsp = (short)kl.num_pixels;
    const short half_h = (height_lsp - 1) / 2;
    const short half_w = (length_lsp - 1) / 2;
    const float mid_x = (float)(0.5 * (kl.s_oct_x + kl.e_oct_x));
    const float mid_y = (float)(0.5 * (kl.s_oct_y + kl.e_oct_y));
    // `cos(float)` inside namespace cv: the double overload of <math.h>, result stored to float (determinism rule: det_cos)
    const float dl0 = libm ? (float)std::cos((double)kl.angle) : (float)det_cos((double)kl.angle);
    const float dl1 = libm ? (float)std::sin((double)kl.angle) : (float)det_sin((double)kl.angle);
    const float do0 = -dl1, do1 = dl0;
    float scx0 = -dl0 * half_w + dl1 * half_h + mid_x;
    float scy0 = -dl1 * half_w - dl0 * half_h + mid_y;
    for (short hid = 0; hid < height_lsp; ++hid) {
        float scx = scx0, scy = scy0;
        float pl = 0, nl = 0, po = 0, no = 0;
        for (short wid = 0; wid < length_lsp; ++wid) {
            short t = (short)std::round(scx);
            const short xc = (t < 0) ? 0 : (t > image_w) ? image_w : t;
            t = (short)std::round(scy);
            const short yc = (t < 0) ? 0 : (t > image_h) ? image_h : t;
            const short dx = dximg[(size_t)yc * w + xc], dy = dyimg[(size_t)yc * w + xc];
            const float gdl = dx * dl0 + dy * dl1;
            const float gdo = dx * do0 + dy * do1;
            if (gdl > 0) pl += gdl; else nl -= gdl;
            if (gdo > 0) po += gdo; else no -= gdo;
            scx += dl0;
            scy += dl1;
        }
        scx0 -= dl1;
        scy0 += dl0;
        float coef = gg[hid];
        pl = coef * pl;
        nl = coef * nl;
        const float pl2 = pl * pl, nl2 = nl * nl;
        po = coef * po;
        no = coef * no;
        const float po2 = po * po, no2 = no * no;
        auto add = [&](int b, float c) {
            band[0][b] += c * pl;
            band[1][b] += c * nl;
            band[2][b] += c * c * pl2;
            band[3][b] += c * c * nl2;
            band[4][b] += c * po;
            band[5][b] += c * no;
            band[6][b] += c * c * po2;
            band[7][b] += c * c * no2;
        };
        short b = (short)(hid / kBandWidth);
        add(b, gl[hid % kBandWidth + kBandWidth]);
        --b;
        if (b >= 0) add(b, gl[hid % kBandWidth + 2 * kBandWidth]);
        b = b + 2;
        if (b < kBands) add(b, gl[hid % kBandWidth]);
    }
    const float inv_n2 = (float)(1.0 / (kBandWidth * 2.0)), inv_n3 = (float)(1.0 / (kBandWidth * 3.0));
    for (int b = 0; b < kBands; ++b) {
        const float inv_n = (b == 0 || b == kBands - 1) ? inv_n2 : inv_n3;
        float *d = des + b * 8;
        float t = band[0][b] * inv_n;
        d[0] = t;
        d[4] = std::sqrt(band[2][b] * inv_n - t * t);
        t = band[1][b] * inv_n;
        d[1] = t;
        d[5] = std::sqrt(band[3][b] * inv_n - t * t);
        t = band[4][b] * inv_n;
        d[2] = t;
        d[6] = std::sqrt(band[6][b] * inv_n - t * t);
        t = band[5][b] * inv_n;
        d[3] = t;
        d[7] = std::sqrt(band[7][b] * inv_n - t * t);
    }
    float tm = 0, ts = 0;
    for (int b = 0; b < kBands; ++b) {
        const float *d = des + b * 8;
        tm += d[0] * d[0];
        tm += d[1] * d[1];
        tm += d[2] * d[2];
        tm += d[3] * d[3];
        ts += d[4] * d[4];
        ts += d[5] * d[5];
        ts += d[6] * d[6];
        ts += d[7] * d[7];
    }
    tm = 1 / std::sqrt(tm);
    ts = 1 / std::sqrt(ts);
    for (int b = 0; b < kBands; ++b) {
        float *d = des + b * 8;
        for (int j = 0; j < 4; ++j) d[j] = d[j] * tm;
        for (int j = 4; j < 8; ++j) d[j] = d[j] * ts;
    }
    for (int i = 0; i < kBands * 8; ++i)
        if (des[i] > 0.4) des[i] = (float)0.4;
    float t = 0;
    for (int i = 0; i < kBands * 8; ++i) t += des[i] * des[i];
    t = 1 / std::sqrt(t);
    for (int i = 0; i < kBands * 8; ++i) des[i] = des[i] * t;
}

void lbd_gradients(const uint8_t *img, int w, int h, int step, std::vector<int16_t> &dx, std::vector<int16_t> &dy) {
    std::vector<uint8_t> g((size_t)w * h);
    blur_q8(img, w, h, step, g.data(), w, kGauss5, 5);
    dx.assign((size_t)w * h, 0);
    dy.assign((size_t)w * h, 0);
    for (int y = 0; y < h; ++y) {
        const uint8_t *r0 = &g[(size_t)reflect101(y - 1, h) * w], *r1 = &g[(size_t)y * w], *r2 = &g[(size_t)reflect101(y + 1, h) * w];
        for (int x = 0; x < w; ++x) {
            const int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w);
            dx[(size_t)y * w + x] = (int16_t)((r0[xp] - r0[xm]) + 2 * (r1[xp] - r1[xm]) + (r2[xp] - r2[xm]));
            dy[(size_t)y * w + x] = (int16_t)((r2[xm] - r0[xm]) + 2 * (r2[x] - r0[x]) + (r2[xp] - r0[xp]));
        }
    }
}

void lbd_compute(const uint8_t *img, int w, int h, int step, const orc_keyline *kl, int n, bool libm, uint8_t *desc,
                 float *desc_float) {
    std::vector<int16_t> dx, dy;
    lbd_gradients(img, w, h, step, dx, dy);
    float gl[kBandWidth * 3], gg[kBands * kBandWidth];
    lbd_weights(gl, gg);
    for (int i = 0; i < n; ++i) {
        float des[kBands * 8];
        lbd_one(dx.data(), dy.data(), w, h, kl[i], libm, gl, gg, des);
        if (desc_float) std::memcpy(desc_float + (size_t)i * 72, des, sizeof(des));
        // binary_descriptor_custom.cpp:398-408, 642-646: byte c, bit b = des[8*i+b] > des[8*j+b]
        for (int c = 0; c < 32; ++c) {
            const float *f1 = des + 8 * kCombinations[c][0], *f2 = des + 8 * kCombinations[c][1];
            uint8_t r = 0;
            for (int b = 0; b < 8; ++b)
                if (f1[b] > f2[b]) r = (uint8_t)(r + (1u << b));
            desc[(size_t)i * 32 + c] = r;
        }
    }
}

}  // namespace

extern "C" {

void orc_lsd_scaled_image(const uint8_t *img, int w, int h, int step, uint8_t *out) {
    std::vector<uint8_t> s;
    int sw, sh;
    scaled_image(img, w, h, step, s, sw, sh);
    std::memcpy(out, s.data(), s.size());
}

int orc_lsd_ll_angle(const uint8_t *scaled, int w, int h, const orc_lsd_config *cfg, float *angle_deg, int32_t *grad_sq,
                     int32_t *bins, int32_t *order) {
    Lsd L;
    L.w = w;
    L.h = h;
    L.cfg = {cfg->seed_order != 0, cfg->libm_float != 0, cfg->sum_order != 0};
    const double rho = kQuant / std::sin(kPi * kAngTh / 180);
    if (bins) std::fill(bins, bins + (size_t)w * h, -1);
    L.ll_angle(scaled, rho, kBins, bins);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const size_t a = (size_t)y * w + x;
            if (angle_deg) angle_deg[a] = L.angles[a] == kNotDef ? -1024.f : (float)(L.angles[a] / kDegToRads);
            if (grad_sq) {
                if (x < w - 1 && y < h - 1) {
                    const int DA = scaled[a + w + 1] - scaled[a], BC = scaled[a + 1] - scaled[a + w];
                    grad_sq[a] = (DA + BC) * (DA + BC) + (DA - BC) * (DA - BC);
                } else
                    grad_sq[a] = 0;
            }
        }
    if (order)
        for (size_t i = 0; i < L.ordered.size(); ++i) order[i] = L.ordered[i].y * w + L.ordered[i].x;
    return (int)L.ordered.size();
}

/* debug: one 11-int record per seed the sequential detector processes (see lsd_detect); returns the record count */
int orc_debug_lsd_trace(const uint8_t *img, int w, int h, int step, const orc_lsd_config *cfg, int32_t *out, int cap_records) {
    std::vector<float> segs;
    std::vector<int32_t> tr;
    lsd_detect(img, w, h, step, cfg, segs, &tr);
    const int n = (int)(tr.size() / 11);
    if (n > cap_records) return -n;
    std::memcpy(out, tr.data(), tr.size() * sizeof(int32_t));
    return n;
}

int orc_lsd_detect(const uint8_t *img, int w, int h, int step, const orc_lsd_config *cfg, float *segments, int cap) {
    std::vector<float> segs;
    const int n = lsd_detect(img, w, h, step, cfg, segs);
    if (n > cap) return -n;
    std::memcpy(segments, segs.data(), segs.size() * sizeof(float));
    return n;
}

int orc_lsd_keylines(const uint8_t *img, int w, int h, int step, const orc_lsd_config *cfg, double min_length,
                     orc_keyline *out, int cap) {
    std::vector<float> segs;
    lsd_detect(img, w, h, step, cfg, segs);
    std::vector<orc_keyline> kls;
    const int n = make_keylines(segs, w, h, cfg, min_length, kls);
    if (n > cap) return -n;
    std::memcpy(out, kls.data(), kls.size() * sizeof(orc_keyline));
    return n;
}

void orc_lbd_gradients(const uint8_t *img, int w, int h, int step, int16_t *dx, int16_t *dy) {
    std::vector<int16_t> vx, vy;
    lbd_gradients(img, w, h, step, vx, vy);
    std::memcpy(dx, vx.data(), vx.size() * 2);
    std::memcpy(dy, vy.data(), vy.size() * 2);
}

void orc_lbd_compute(const uint8_t *img, int w, int h, int step, const orc_keyline *kl, int n, int libm_float,
                     uint8_t *desc, float *desc_float) {
    lbd_compute(img, w, h, step, kl, n, libm_float != 0, desc, desc_float);
}

int orc_line_extract(const uint8_t *img, int w, int h, int step, const orc_lsd_config *cfg, orc_keyline *kl_out,
                     uint8_t *lbd_out, double *fn_out, int cap) {
    // line_extractor.cc:103 remap with the identity map == copy (SURVEY Appendix A.6); :122 min_length = 0.125 * min(w, h)
    std::vector<float> segs;
    lsd_detect(img, w, h, step, cfg, segs);
    std::vector<orc_keyline> kls;
    const double min_length = 0.125 * std::min(w, h);
    make_keylines(segs, w, h, cfg, min_length, kls);
    if (kls.empty()) return 0;  // computeImpl prints "keypoint list is empty" and returns (binary_descriptor_custom.cpp:537-541)
    std::vector<uint8_t> desc(kls.size() * 32);
    lbd_compute(img, w, h, step, kls.data(), (int)kls.size(), cfg->libm_float != 0, desc.data(), nullptr);
    int n = 0;
    for (size_t i = 0; i < kls.size(); ++i)
        if (kls[i].octave == 0 && kls[i].line_length >= 60) ++n;  // line_extractor.cc:134-141
    if (n > cap) return -n;
    n = 0;
    for (size_t i = 0; i < kls.size(); ++i) {
        if (!(kls[i].octave == 0 && kls[i].line_length >= 60)) continue;
        kl_out[n] = kls[i];
        std::memcpy(lbd_out + (size_t)n * 32, &desc[i * 32], 32);
        // line_extractor.cc:147-159: l = sp x ep / ||(l0, l1)||  (doubles)
        const double sx = kls[i].start_x, sy = kls[i].start_y, ex = kls[i].end_x, ey = kls[i].end_y;
        const double l0 = sy * 1.0 - 1.0 * ey, l1 = 1.0 * ex - sx * 1.0, l2 = sx * ey - sy * ex;
        const double nrm = std::sqrt(l0 * l0 + l1 * l1);
        fn_out[3 * n] = l0 / nrm;
        fn_out[3 * n + 1] = l1 / nrm;
        fn_out[3 * n + 2] = l2 / nrm;
        ++n;
    }
    return n;
}

}  // extern "C"

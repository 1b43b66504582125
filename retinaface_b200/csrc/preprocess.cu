// preprocess.cu -- see preprocess.cuh.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <type_traits>

#include "preprocess.cuh"
#include "warp.cuh"

namespace rf {

void letterbox_geometry(int w, int h, int net_w, int net_h, int *dw, int *dh, double *scale) {
    // RetinaFace.cpp:587-591: float sw = 1.0*cols/inputW, sh = 1.0*rows/inputH; scale = max(sw, sh, 1)
    float sw = (float)(1.0 * w / net_w), sh = (float)(1.0 * h / net_h);
    float sc = sw > sh ? sw : sh;
    sc = sc > 1.0f ? sc : 1.0f;
    if (sc > 1.0f) {
        double f = (double)(1 / sc);              // cv::resize(..., fx = 1/scale (float), fy = same)
        *dw = (int)std::nearbyint(w * f);         // saturate_cast<int>(double): round half to even
        *dh = (int)std::nearbyint(h * f);
        *scale = 1.0 / f;                         // resize.cpp: scale_x = 1. / inv_scale_x
    } else {
        *dw = w; *dh = h; *scale = 1.0;
    }
    if (*dw > net_w) *dw = net_w;                 // copyMakeBorder would assert; clamp instead
    if (*dh > net_h) *dh = net_h;
}

namespace {

struct Tap { int s0, s1, a0, a1; };

// OpenCV resizeGeneric_ linear coefficient of one destination coordinate (resize.cpp, INTER_LINEAR).
// Horizontal taps zero the fraction at the borders (xmin/xmax handling); vertical taps keep the
// fraction and clamp the source ROW indices instead (resizeGeneric_Invoker: sy = clip(sy0 + k, 0, h)),
// which differs by one count after the truncating vertical pass.
template <bool HORIZONTAL>
__device__ __forceinline__ Tap tap_of(int d, int sn, double scale) {
    float fx = (float)((d + 0.5) * scale - 0.5);
    int s = (int)floorf(fx);
    fx -= (float)s;
    if (HORIZONTAL) {
        if (s < 0) { fx = 0.f; s = 0; }
        if (s >= sn - 1) { fx = 0.f; s = sn - 1; }
    }
    Tap t;
    t.s0 = min(max(s, 0), sn - 1);
    t.s1 = min(max(s + 1, 0), sn - 1);
    t.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f));   // saturate_cast<short>(cbuf*INTER_RESIZE_COEF_SCALE)
    t.a1 = __float2int_rn(__fmul_rn(fx, 2048.f));
    return t;
}

// One launch letter-boxes up to LB_MAX_IMAGES images (LB_MAX_FRAMES frames): blockIdx.z = image, blockIdx.y = output row, a
// thread = 4 consecutive output pixels = 12 bytes = three aligned 32-bit stores (net_w is a multiple of 32, so rows start 4-byte
// aligned).  Per image (LbItemT): the source, dst = net_h x net_w x 3, the source size, the size of the resized image inside
// the output (top-left, the rest is 0), the source pixels per output pixel.
template <typename Src> constexpr int lb_limit() { return std::is_same<Src, BgrRows>::value ? LB_MAX_IMAGES : LB_MAX_FRAMES; }
template <typename Src>
struct LbBatch { LbItemT<Src> img[lb_limit<Src>()]; };
static_assert(sizeof(LbItemT<BgrRows>) == 56, "64 BGR items per launch rely on the 56-byte item");
static_assert(sizeof(LbBatch<BgrRows>) + 8 <= 4096 && sizeof(LbBatch<YuvPlanes>) + 8 <= 4096,
              "letter-box chunk exceeds the classic 4 KB kernel parameter space");

// BGR of stored pixel (x, y): u8 BGR rows, or a YUV 4:2:0 frame converted on the fly
__device__ __forceinline__ void src_pixel(const BgrRows &src, int x, int y, int v[3]) {
    const uint8_t *p = src.p + (size_t)y * src.pitch + (size_t)x * 3;
    v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
}
__device__ __forceinline__ void src_pixel(const YuvPlanes &src, int x, int y, int v[3]) { yuv_pixel(src, x, y, v); }

// f9: the orientation touches integer tap addresses only.  Every tap position, weight and rounding below is computed in the
// DISPLAYED frame (sw x sh), a displayed column / row is then reflected by the item's LB_FLIP_X / LB_FLIP_Y bit, and the transposed
// instantiation (T) reads displayed (x, y) at stored column y, stored row x -- so the bytes are those of cv::resize(T_o(img)).
template <typename Src> __device__ __forceinline__ int col_of(const LbItemT<Src> &im, int x) { return (im.flip & LB_FLIP_X) ? im.sw - 1 - x : x; }
template <typename Src> __device__ __forceinline__ int row_of(const LbItemT<Src> &im, int y) { return (im.flip & LB_FLIP_Y) ? im.sh - 1 - y : y; }
template <bool T, typename Src>
__device__ __forceinline__ void stored_pixel(const LbItemT<Src> &im, int x, int y, int v[3]) {
    if (T) src_pixel(im.src, y, x, v);
    else src_pixel(im.src, x, y, v);
}

// NPP's NPPI_INTER_SUPER as measured against nppiResizeSqrPixel_8u_C3R (tools/npp_dump.py, oracle/npp_oracle.cu):
// output pixel (x, y) = the coverage-weighted mean of the source rectangle [x / f, (x + 1) / f) x [y / f, (y + 1) / f), the
// resized extent is ceil(w f) x ceil(h f), source samples beyond the image count as ZERO (the last row / column is darker, not
// renormalised), round half up.  Matches NPP byte for byte on 5 of 8 probe shapes and within 1 LSB on < 0.5 % of the bytes of
// the others (NPP's own arithmetic is single precision).
template <bool T, typename Src>
__device__ __forceinline__ void area_pixel(const LbItemT<Src> &im, int x, int y, int out[3]) {
    const double inv = im.scale;
    const double ax = x * inv, bx = (x + 1) * inv, ay = y * inv, by = (y + 1) * inv;
    const int x0 = (int)floor(ax), x1 = min((int)ceil(bx - 1e-12), im.sw), y0 = (int)floor(ay), y1 = min((int)ceil(by - 1e-12), im.sh);
    double acc[3] = {0.0, 0.0, 0.0};
    for (int sy = y0; sy < y1; sy++) {
        const double wy = fmin((double)(sy + 1), by) - fmax((double)sy, ay);
        for (int sx = x0; sx < x1; sx++) {
            const double w = wy * (fmin((double)(sx + 1), bx) - fmax((double)sx, ax));
            int p[3];
            stored_pixel<T>(im, col_of(im, sx), row_of(im, sy), p);
            acc[0] += w * p[0]; acc[1] += w * p[1]; acc[2] += w * p[2];
        }
    }
    const double norm = 1.0 / (inv * inv);
#pragma unroll
    for (int c = 0; c < 3; c++) out[c] = min(max((int)floor(acc[c] * norm + 0.5), 0), 255);
}

template <bool T, typename Src>
__device__ __forceinline__ void linear_pixel(const LbItemT<Src> &im, int x, Tap ty, int out[3]) {
    Tap tx = tap_of<true>(x, im.sw, im.scale);
    tx.s0 = col_of(im, tx.s0); tx.s1 = col_of(im, tx.s1);
    ty.s0 = row_of(im, ty.s0); ty.s1 = row_of(im, ty.s1);
    int p00[3], p01[3], p10[3], p11[3];
    stored_pixel<T>(im, tx.s0, ty.s0, p00); stored_pixel<T>(im, tx.s1, ty.s0, p01);
    stored_pixel<T>(im, tx.s0, ty.s1, p10); stored_pixel<T>(im, tx.s1, ty.s1, p11);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        int h0 = p00[c] * tx.a0 + p01[c] * tx.a1;   // HResizeLinear
        int h1 = p10[c] * tx.a0 + p11[c] * tx.a1;
        int v = (((ty.a0 * (h0 >> 4)) >> 16) + ((ty.a1 * (h1 >> 4)) >> 16) + 2) >> 2;  // VResizeLinear 8u
        out[c] = min(max(v, 0), 255);
    }
}

// cv::resize's INTER_LINEAR at exactly 2x down-scaling in both axes, where OpenCV takes its fast INTER_AREA path instead
// (resize.cpp: `interpolation == INTER_LINEAR && is_area_fast && iscale_x == 2 && iscale_y == 2`): output pixel (x, y) is the mean
// of the source block [2x, 2x + 2) x [2y, 2y + 2).  A whole block rounds as the bilinear taps would, (sum + 2) >> 2; a block cut by
// the far edge of a side of 3 mod 4 (whose halved size rounds up) averages the pixels it has, rounded half to even.
template <bool T, typename Src>
__device__ __forceinline__ void half_pixel(const LbItemT<Src> &im, int x, int y, int out[3]) {
    const int nx = min(2, im.sw - 2 * x), ny = min(2, im.sh - 2 * y);
    int acc[3] = {0, 0, 0};
    for (int sy = 0; sy < ny; sy++)
        for (int sx = 0; sx < nx; sx++) {
            int p[3];
            stored_pixel<T>(im, col_of(im, 2 * x + sx), row_of(im, 2 * y + sy), p);
            acc[0] += p[0]; acc[1] += p[1]; acc[2] += p[2];
        }
    const int cnt = nx * ny;
#pragma unroll
    for (int c = 0; c < 3; c++) out[c] = cnt == 4 ? (acc[c] + 2) >> 2 : __float2int_rn(__fdiv_rn((float)acc[c], (float)cnt));
}

// Pixel (x, y) of the resized displayed image (inside dw x dh); ty: the vertical bilinear tap of row y (bilinear items only).
template <bool T, typename Src>
__device__ __forceinline__ void lb_pixel(const LbItemT<Src> &im, int x, int y, const Tap &ty, int v[3]) {
    if (im.identity) {
        stored_pixel<T>(im, col_of(im, x), row_of(im, y), v);
    } else if (im.area == LB_HALF_AREA) {
        half_pixel<T>(im, x, y, v);
    } else if (im.area) {
        area_pixel<T>(im, x, y, v);
    } else {
        linear_pixel<T>(im, x, ty, v);
    }
}

template <typename Src>
__global__ void __launch_bounds__(128) k_letterbox_batch(const __grid_constant__ LbBatch<Src> B, int net_w, int net_h) {
    const LbItemT<Src> &im = B.img[blockIdx.z];
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x4 >= net_w) return;
    // pixel (x4 + k, blockIdx.y) of the output is pixel (x, y) of the resized image (a tile's origin; 0 for the letter-box)
    const int y = blockIdx.y + im.y0;
    unsigned char px[12];
    const bool row_in = y < im.dh;
    Tap ty{};
    if (row_in && !im.identity && !im.area) ty = tap_of<false>(y, im.sh, im.scale);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int x = x4 + k + im.x0;
        int v[3] = {0, 0, 0};
        // flip bits: the view is the letter-box of the mirrored / upside-down image -- every source column / row index is reflected,
        // the taps are those of the reflected image (== cv::resize(cv::flip(img, ...)) bit for bit)
        if (row_in && x < im.dw) lb_pixel<false>(im, x, y, ty, v);
        px[3 * k] = (unsigned char)v[0]; px[3 * k + 1] = (unsigned char)v[1]; px[3 * k + 2] = (unsigned char)v[2];
    }
    uint32_t *o = reinterpret_cast<uint32_t *>(im.dst + ((size_t)blockIdx.y * net_w + x4) * 3);
    o[0] = px[0] | (px[1] << 8) | (px[2] << 16) | ((uint32_t)px[3] << 24);
    o[1] = px[4] | (px[5] << 8) | (px[6] << 16) | ((uint32_t)px[7] << 24);
    o[2] = px[8] | (px[9] << 8) | (px[10] << 16) | ((uint32_t)px[11] << 24);
}

// f9, the transposed orientations (LB_TRANSPOSE: EXIF 5..8).  Consecutive output pixels of a row read consecutive stored ROWS, so a
// row-per-thread gather would touch one 3-byte pixel per stored row per lane.  Instead a CTA computes one 32 x 32 block of the output:
// lane l of each warp takes output row by + l, so the 32 lanes of a warp read 32 consecutive pixels of one stored row, and the warps
// step over the block's columns.  The block goes through shared memory (rows padded to 25 words: the lanes' byte writes fall in
// distinct banks) and leaves as whole output rows, 24 consecutive 32-bit words each.
constexpr int LBT_SIDE = 32, LBT_THREADS = 128, LBT_ROW_WORDS = 25;
template <typename Src>
__global__ void __launch_bounds__(LBT_THREADS) k_letterbox_transposed(const __grid_constant__ LbBatch<Src> B, int net_w, int net_h) {
    __shared__ uint32_t s_blk[LBT_SIDE * LBT_ROW_WORDS];
    const LbItemT<Src> &im = B.img[blockIdx.z];
    unsigned char *sb = reinterpret_cast<unsigned char *>(s_blk);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int bx = blockIdx.x * LBT_SIDE, by = blockIdx.y * LBT_SIDE;
    const int oy = by + lane, y = oy + im.y0;
    const bool row_in = oy < net_h && y < im.dh;
    Tap ty{};
    if (row_in && !im.identity && !im.area) ty = tap_of<false>(y, im.sh, im.scale);
    for (int c = warp; c < LBT_SIDE; c += LBT_THREADS / 32) {
        const int x = bx + c + im.x0;
        int v[3] = {0, 0, 0};
        if (row_in && x < im.dw) lb_pixel<true>(im, x, y, ty, v);
        unsigned char *d = sb + lane * (LBT_ROW_WORDS * 4) + 3 * c;
        d[0] = (unsigned char)v[0]; d[1] = (unsigned char)v[1]; d[2] = (unsigned char)v[2];
    }
    __syncthreads();
    constexpr int kWords = LBT_SIDE * 3 / 4;      // 24 words per output row of the block
    for (int k = threadIdx.x; k < LBT_SIDE * kWords; k += LBT_THREADS) {
        const int r = k / kWords, w = k - r * kWords;
        if (by + r >= net_h) break;
        uint32_t *o = reinterpret_cast<uint32_t *>(im.dst + ((size_t)(by + r) * net_w + bx) * 3);
        o[w] = s_blk[r * LBT_ROW_WORDS + w];
    }
}

}  // namespace

void letterbox_geometry_npp(int w, int h, int net_w, int net_h, int *dw, int *dh, double *scale) {
    // resizeconvertion.cu:298-303: factor = min(dstW / srcW, dstH / srcH), clamped to <= 1 (never up-scaled)
    const double fx = (double)net_w / w, fy = (double)net_h / h;
    double f = fx < fy ? fx : fy;
    if (f >= 1.0) { *dw = std::min(w, net_w); *dh = std::min(h, net_h); *scale = 1.0; return; }
    *dw = std::min((int)std::ceil(w * f - 1e-9), net_w);
    *dh = std::min((int)std::ceil(h * f - 1e-9), net_h);
    *scale = 1.0 / f;
}

float letterbox_map_back(int w, int h, int box_w, int box_h) {
    const float sw = (float)(1.0 * w / box_w), sh = (float)(1.0 * h / box_h);
    const float sc = sw > sh ? sw : sh;
    return sc > 1.0f ? sc : 1.0f;
}

template <typename Src>
float letterbox_fill(LbItemT<Src> &it, typename LbItemT<Src>::Source src, int w, int h, uint8_t *dst, int box_w, int box_h, int flip, int area) {
    it.src = src; it.dst = dst; it.sw = w; it.sh = h; it.flip = flip; it.area = area;
    it.x0 = it.y0 = 0;
    if (area) letterbox_geometry_npp(w, h, box_w, box_h, &it.dw, &it.dh, &it.scale);
    else letterbox_geometry(w, h, box_w, box_h, &it.dw, &it.dh, &it.scale);
    it.identity = it.scale == 1.0 ? 1 : 0;
    if (it.identity) it.area = 0;
    else if (!area && it.scale == 2.0) it.area = LB_HALF_AREA;   // cv::resize's own branch at exactly 2x, as tile_fill takes it
    return letterbox_map_back(w, h, box_w, box_h);
}

// ---- f7 tiles -------------------------------------------------------------------------------------------------------------------
namespace {
constexpr int TILE_MAX_SIDE = 16384;   // largest resized level side
static_assert(TILE_MAX_SIDE <= 32767, "tile origins travel as int16_t (LbItemT)");

// The tiles of one axis of a level of size S: origins and the half-open ownership cores (see rf_b200.h).
struct AxisTiles { std::vector<int> origin, own0, own1; };
AxisTiles axis_tiles(int S, int T, int o) {
    AxisTiles a;
    const int k = S <= T ? 1 : (S - o + (T - o) - 1) / (T - o);
    for (int i = 0; i < k; i++) a.origin.push_back(S <= T ? 0 : std::min(i * (T - o), S - T));
    for (int i = 0; i < k; i++) {
        a.own0.push_back(i == 0 ? 0 : a.own1[i - 1]);
        // the last core ends at the far edge of the last tile: S when the axis is tiled, T (the padding included) when one tile
        // holds the whole axis
        a.own1.push_back(i == k - 1 ? a.origin[i] + T : (a.origin[i + 1] + a.origin[i] + T) / 2);
    }
    return a;
}

// saturate_cast<int>(side * s): cv::resize's size of a level (round half to even)
int level_side(int side, double s) { return (int)std::nearbyint(side * s); }

// The refusals of an rf_tiling that hold whatever the image size, each with its message.
bool bad_nlevels(int nlevels, std::string &msg) {
    if (nlevels >= 0 && nlevels <= RF_MAX_TILE_LEVELS) return false;
    msg = "nlevels " + std::to_string(nlevels) + ", must be in [0, " + std::to_string(RF_MAX_TILE_LEVELS) + "]";
    return true;
}
bool bad_overlap(int net_w, int net_h, const rf_tiling *t, std::string &msg) {
    const int o_max = std::min(net_w, net_h) / 2;
    const int o = t && t->overlap ? t->overlap : 64;
    if (o >= 16 && o <= o_max) return false;
    char buf[128];
    snprintf(buf, sizeof buf, "overlap %d, must be 0 (64) or in [16, %d]", t ? t->overlap : 0, o_max);
    msg = buf;
    return true;
}
bool bad_scale(size_t l, float s, std::string &msg) {
    if (s >= 0.f && std::isfinite(s)) return false;
    char buf[128];
    snprintf(buf, sizeof buf, "level %zu: scale %g, must be finite and >= 0", l, (double)s);
    msg = buf;
    return true;
}
}  // namespace

int tiling_check(int net_w, int net_h, const rf_tiling *t, std::string *err) {
    std::string msg;
    bool bad = bad_nlevels(t ? t->nlevels : 0, msg) || bad_overlap(net_w, net_h, t, msg);
    for (int l = 0; !bad && t && t->levels && l < t->nlevels; l++) bad = bad_scale(l, t->levels[l].scale, msg);
    if (bad && err) *err = msg;
    return bad ? RF_ERR_INVALID_ARG : RF_OK;
}

int tile_layout(int net_w, int net_h, int w, int h, const rf_tiling *t, std::vector<rf_tile> &out, std::string *err) {
    out.clear();
    auto bad = [&](int status, const std::string &msg) { if (err) *err = msg; out.clear(); return status; };
    char buf[256];
    std::string msg;
    if (net_w <= 0 || net_h <= 0 || w <= 0 || h <= 0) return bad(RF_ERR_INVALID_ARG, "image and network sizes must be positive");
    const int nlevels = t ? t->nlevels : 0;
    if (bad_nlevels(nlevels, msg)) return bad(RF_ERR_INVALID_ARG, msg);
    if (nlevels > 0 && !t->levels) return bad(RF_ERR_INVALID_ARG, "levels is NULL");
    const int o = t && t->overlap ? t->overlap : 64;
    if (bad_overlap(net_w, net_h, t, msg)) return bad(RF_ERR_INVALID_ARG, msg);
    std::vector<rf_tile_level> levels;
    if (nlevels > 0) {
        levels.assign(t->levels, t->levels + nlevels);
    } else {
        // the default pyramid: 1, 1/2, 1/4, ... while the level does not fit in one tile, then the fitted level
        for (float s = 1.f; level_side(w, s) > net_w || level_side(h, s) > net_h; s *= 0.5f) levels.push_back(rf_tile_level{s, 0});
        levels.push_back(rf_tile_level{0.f, 0});
    }
    for (size_t l = 0; l < levels.size(); l++) {
        const float s = levels[l].scale;
        if (bad_scale(l, s, msg)) return bad(RF_ERR_INVALID_ARG, msg);
        int sw, sh;
        float map_back;
        if (s == 0.f) {       // the fitted level: rf_detect_batch's letter-box
            double inv;
            letterbox_geometry(w, h, net_w, net_h, &sw, &sh, &inv);
            map_back = letterbox_map_back(w, h, net_w, net_h);
        } else {
            sw = level_side(w, s);
            sh = level_side(h, s);
            map_back = (float)(1.0 / (double)s);
        }
        if (sw < 1 || sh < 1 || sw > TILE_MAX_SIDE || sh > TILE_MAX_SIDE) {
            snprintf(buf, sizeof buf, "level %zu: scale %g resizes %dx%d to %dx%d; each side must be in [1, %d]", l, (double)s, w, h, sw, sh,
                     TILE_MAX_SIDE);
            return bad(RF_ERR_INVALID_ARG, buf);
        }
        const AxisTiles ax = axis_tiles(sw, net_w, o), ay = axis_tiles(sh, net_h, o);
        if (out.size() + ax.origin.size() * ay.origin.size() > (size_t)RF_MAX_TILES) {
            snprintf(buf, sizeof buf, "the layout of a %dx%d image has more than RF_MAX_TILES = %d tiles", w, h, RF_MAX_TILES);
            return bad(RF_ERR_CAPACITY, buf);
        }
        for (size_t j = 0; j < ay.origin.size(); j++)
            for (size_t i = 0; i < ax.origin.size(); i++) {
                rf_tile tl{};
                tl.level = (int)l;
                tl.flip = levels[l].flip ? 1 : 0;
                tl.scaled_w = sw; tl.scaled_h = sh;
                tl.x0 = ax.origin[i]; tl.y0 = ay.origin[j];
                tl.own_x0 = ax.own0[i]; tl.own_x1 = ax.own1[i];
                tl.own_y0 = ay.own0[j]; tl.own_y1 = ay.own1[j];
                tl.shared_sides = (i > 0 ? RF_TILE_SIDE_LEFT : 0) | (j > 0 ? RF_TILE_SIDE_TOP : 0) |
                                  (i + 1 < ax.origin.size() ? RF_TILE_SIDE_RIGHT : 0) | (j + 1 < ay.origin.size() ? RF_TILE_SIDE_BOTTOM : 0);
                tl.scale = s;
                tl.map_back = map_back;
                out.push_back(tl);
            }
    }
    return RF_OK;
}

template <typename Src>
void tile_fill(LbItemT<Src> &it, typename LbItemT<Src>::Source src, int w, int h, int bits, uint8_t *dst, int net_w, int net_h,
               const rf_tile &tile) {
    // the LB bits act on displayed coordinates before the transpose: mirroring the displayed image flips displayed x
    const int flip = bits ^ (tile.flip ? LB_FLIP_X : 0);
    if (tile.scale == 0.f) {          // the fitted level: the letter-box itself
        letterbox_fill(it, src, w, h, dst, net_w, net_h, flip, 0);
        return;
    }
    it.src = src; it.dst = dst; it.sw = w; it.sh = h; it.flip = flip;
    it.dw = tile.scaled_w; it.dh = tile.scaled_h;
    it.scale = 1.0 / (double)tile.scale;     // cv::resize: scale_x = 1. / inv_scale_x
    it.identity = it.scale == 1.0 ? 1 : 0;
    it.area = it.scale == 2.0 ? LB_HALF_AREA : 0;
    it.x0 = (int16_t)tile.x0; it.y0 = (int16_t)tile.y0;
}

template <typename Src>
cudaError_t launch_letterbox_batch(const LbItemT<Src> *items, int n, int net_w, int net_h, cudaStream_t s) {
    constexpr int kMax = lb_limit<Src>();
    for (int i0 = 0; i0 < n; i0 += kMax) {
        const int m = std::min(kMax, n - i0);
        // a chunk that mixes orientations is two launches: the upright / reflected items, then the transposed ones
        LbBatch<Src> B{}, Bt{};
        int nb = 0, nt = 0;
        for (int i = 0; i < m; i++) {
            const LbItemT<Src> &it = items[i0 + i];
            if (it.flip & LB_TRANSPOSE) Bt.img[nt++] = it;
            else B.img[nb++] = it;
        }
        if (nb) k_letterbox_batch<Src><<<dim3((net_w / 4 + 127) / 128, net_h, nb), 128, 0, s>>>(B, net_w, net_h);
        if (nt) k_letterbox_transposed<Src><<<dim3(net_w / LBT_SIDE, (net_h + LBT_SIDE - 1) / LBT_SIDE, nt), LBT_THREADS, 0, s>>>(Bt, net_w, net_h);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- f23 rotated views ------------------------------------------------------------------------------------------------------------
RotatedGeometry rotated_geometry(float angle, int w, int h, int box_w, int box_h) {
    RotatedGeometry g{};
    double a = std::fmod((double)angle, 360.0);
    if (a < 0.0) a += 360.0;
    if (a == 360.0) a = 0.0;      // a negative angle above -2^-45 rounds up to a whole turn
    if (a == 0.0 || a == 90.0 || a == 180.0 || a == 270.0) {
        g.orientation = a == 0.0 ? 1 : a == 90.0 ? 8 : a == 180.0 ? 3 : 6;
        return g;
    }
    const double r = a * (M_PI / 180.0), c = std::cos(r), s = std::sin(r);
    const double W = w, H = h;
    const double wr = std::fabs(c) * W + std::fabs(s) * H, hr = std::fabs(s) * W + std::fabs(c) * H;
    double f = 1.0;
    f = std::min(f, box_w / wr);
    f = std::min(f, box_h / hr);
    g.f = f;
    g.M[0] = f * c; g.M[1] = f * s; g.M[3] = -(f * s); g.M[4] = f * c;
    const double cx = (W - 1.0) / 2.0, cy = (H - 1.0) / 2.0;
    g.M[2] = (f * wr - 1.0) / 2.0 - (g.M[0] * cx + g.M[1] * cy);
    g.M[5] = (f * hr - 1.0) / 2.0 - (g.M[3] * cx + g.M[4] * cy);
    invert_affine(g.M, g.iM);
    return g;
}

namespace {
// A CTA computes WARP_BAND rows of WARP_SPAN columns of one view (short bands: many CTAs, so that the gathers' latency overlaps): it tabulates OpenCV's per-column (adelta, bdelta) and per-row
// (X0, Y0) fixed-point terms in shared memory as k_align_faces does, so every pixel costs integer arithmetic only, and each thread
// makes 4 consecutive pixels of a row, stored as three aligned 32-bit words (net_w is a multiple of 32).  Per row the CTA also bounds
// the columns whose taps can reach the image; the quads outside that span are zero and gather nothing.
constexpr int WARP_THREADS = 128, WARP_BAND = 2, WARP_SPAN = WARP_THREADS * 4;
template <typename Src>
struct WarpBatch { WarpItemT<Src> v[WARP_MAX_VIEWS]; };
// f25: the oriented launch's items and their LB_* bits
template <typename Src>
struct WarpBatchO { WarpItemT<Src> v[WARP_MAX_VIEWS]; int bits[WARP_MAX_VIEWS]; };
template <typename Src, bool ORIENTED> using WarpBatchT = typename std::conditional<ORIENTED, WarpBatchO<Src>, WarpBatch<Src>>::type;
static_assert(sizeof(WarpBatch<BgrRows>) + 8 <= 4096, "warp launch exceeds the classic 4 KB kernel parameter space");
static_assert(sizeof(WarpItemT<YuvPlanes>) == 104 && sizeof(WarpBatch<YuvPlanes>) + 8 <= 4096,
              "YUV warp launch exceeds the classic 4 KB kernel parameter space");
static_assert(sizeof(WarpBatchO<YuvPlanes>) + 8 <= 4096, "oriented YUV warp launch exceeds the classic 4 KB kernel parameter space");

// [lo, hi] of the x with a x + b in [-2, n + 1]: the fixed-point source coordinate is within 1/16 pixel of a x + b, and a pixel has a
// tap in [0, n) only if that coordinate is in [-1, n), so the bound keeps a pixel of margin
__device__ __forceinline__ void footprint(double a, double b, int n, double &lo, double &hi) {
    if (fabs(a) < 1e-12) {
        const bool in = b >= -2.0 && b <= n + 1.0;
        lo = in ? -INFINITY : INFINITY;
        hi = in ? INFINITY : -INFINITY;
        return;
    }
    const double t0 = (-2.0 - b) / a, t1 = (n + 1.0 - b) / a;
    lo = fmin(t0, t1);
    hi = fmax(t0, t1);
}

// ORIENTED (f25): item z reads the displayed image of its stored source under bits[z] (its w x h displayed), f9's oriented taps.
template <typename Src, bool ORIENTED>
__global__ void __launch_bounds__(WARP_THREADS) k_letterbox_warp(const __grid_constant__ WarpBatchT<Src, ORIENTED> B, int net_w, int net_h) {
    __shared__ int s_ax[WARP_SPAN], s_bx[WARP_SPAN], s_x0[WARP_BAND], s_y0[WARP_BAND], s_lo[WARP_BAND], s_hi[WARP_BAND];
    const WarpItemT<Src> &it = B.v[blockIdx.z];
    const int xb = blockIdx.x * WARP_SPAN, yb = blockIdx.y * WARP_BAND;
    const double i0 = it.im[0], i1 = it.im[1], i2 = it.im[2], i3 = it.im[3], i4 = it.im[4], i5 = it.im[5];
    for (int k = threadIdx.x; k < WARP_SPAN; k += WARP_THREADS) {
        const int x = xb + k;
        s_ax[k] = __double2int_rn(i0 * x * 1024.0);
        s_bx[k] = __double2int_rn(i3 * x * 1024.0);
    }
    if (threadIdx.x < WARP_BAND) {
        const int y = yb + threadIdx.x;
        const double bu = i1 * y + i2, bv = i4 * y + i5;
        s_x0[threadIdx.x] = __double2int_rn(bu * 1024.0) + 16;
        s_y0[threadIdx.x] = __double2int_rn(bv * 1024.0) + 16;
        double ulo, uhi, vlo, vhi;
        footprint(i0, bu, it.w, ulo, uhi);
        footprint(i3, bv, it.h, vlo, vhi);
        const double lo = fmax(ulo, vlo), hi = fmin(uhi, vhi);
        const bool any = lo <= hi;
        const double edge = net_w + 1.0;
        s_lo[threadIdx.x] = any ? (int)floor(fmin(fmax(lo, -2.0), edge)) - 1 : net_w + 8;
        s_hi[threadIdx.x] = any ? (int)ceil(fmin(fmax(hi, -2.0), edge)) + 1 : -8;
    }
    __syncthreads();
    const int x4 = xb + threadIdx.x * 4;
    if (x4 >= net_w) return;
    int orient = 0;
    if constexpr (ORIENTED) orient = B.bits[blockIdx.z];
    const AlignImageT<Src> img{it.src, it.w, it.h, 1.f, orient};
    // every gather of the band before any store: a store may alias the source for all the compiler knows, so interleaving them would
    // serialise the rows' gathers
    int v[WARP_BAND][4][3] = {};
#pragma unroll
    for (int r = 0; r < WARP_BAND; r++) {
        if (yb + r >= net_h || x4 + 3 < s_lo[r] || x4 > s_hi[r]) continue;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int c = threadIdx.x * 4 + k;
            sample<ORIENTED>(img, (s_x0[r] + s_ax[c]) >> 5, (s_y0[r] + s_bx[c]) >> 5, v[r][k]);
        }
    }
#pragma unroll
    for (int r = 0; r < WARP_BAND; r++) {
        if (yb + r >= net_h) break;
        const int(*q)[3] = v[r];
        uint32_t *o = reinterpret_cast<uint32_t *>(it.dst + ((size_t)(yb + r) * net_w + x4) * 3);
        o[0] = q[0][0] | (q[0][1] << 8) | (q[0][2] << 16) | ((uint32_t)q[1][0] << 24);
        o[1] = q[1][1] | (q[1][2] << 8) | (q[2][0] << 16) | ((uint32_t)q[2][1] << 24);
        o[2] = q[2][2] | (q[3][0] << 8) | (q[3][1] << 16) | ((uint32_t)q[3][2] << 24);
    }
}
}  // namespace

template <typename Src>
cudaError_t launch_letterbox_warp(const WarpItemT<Src> *items, int n, int net_w, int net_h, cudaStream_t s, const int *bits) {
    const dim3 block(WARP_THREADS);
    for (int i0 = 0; i0 < n; i0 += WARP_MAX_VIEWS) {
        const int m = std::min(WARP_MAX_VIEWS, n - i0);
        const dim3 grid((net_w + WARP_SPAN - 1) / WARP_SPAN, (net_h + WARP_BAND - 1) / WARP_BAND, m);
        if (bits && std::any_of(bits + i0, bits + i0 + m, [](int b) { return b != 0; })) {
            // only the tracker's YUV frames are oriented: no BGR path passes bits, and none is compiled
            if constexpr (std::is_same<Src, YuvPlanes>::value) {
                WarpBatchO<Src> B{};
                for (int i = 0; i < m; i++) {
                    B.v[i] = items[i0 + i];
                    B.bits[i] = bits[i0 + i];
                }
                k_letterbox_warp<Src, true><<<grid, block, 0, s>>>(B, net_w, net_h);
            } else {
                return cudaErrorNotSupported;
            }
        } else {
            WarpBatch<Src> B{};
            for (int i = 0; i < m; i++) B.v[i] = items[i0 + i];
            k_letterbox_warp<Src, false><<<grid, block, 0, s>>>(B, net_w, net_h);
        }
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}
template cudaError_t launch_letterbox_warp<BgrRows>(const WarpItem *, int, int, int, cudaStream_t, const int *);
template cudaError_t launch_letterbox_warp<YuvPlanes>(const WarpYuvItem *, int, int, int, cudaStream_t, const int *);

template float letterbox_fill<BgrRows>(LbItem &, BgrRows, int, int, uint8_t *, int, int, int, int);
template float letterbox_fill<YuvPlanes>(LbYuvItem &, YuvPlanes, int, int, uint8_t *, int, int, int, int);
template cudaError_t launch_letterbox_batch<BgrRows>(const LbItem *, int, int, int, cudaStream_t);
template cudaError_t launch_letterbox_batch<YuvPlanes>(const LbYuvItem *, int, int, int, cudaStream_t);
template void tile_fill<BgrRows>(LbItem &, BgrRows, int, int, int, uint8_t *, int, int, const rf_tile &);
template void tile_fill<YuvPlanes>(LbYuvItem &, YuvPlanes, int, int, int, uint8_t *, int, int, const rf_tile &);

}  // namespace rf

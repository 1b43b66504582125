// align.cu -- see align.cuh.  Compiled with -fmad=false: OpenCV evaluates iM01 * y + iM02 (and the closed-form sums here
// mirror oracle/align.py) as a separate multiply and add, and a contracted FMA can move a coordinate across a 1/1024
// rounding boundary.
#include "align.cuh"

namespace rf {

size_t align_crop_bytes(int crop_w, int crop_h, int format) {
    const size_t px = (size_t)crop_w * crop_h * 3;
    return format == RF_CROP_RGB_F32 ? px * 4 : format == RF_CROP_RGB_F16 ? px * 2 : px;
}

namespace {

// A work item is one band of ALIGN_BAND crop rows of one (image, face) slot: about two pixel quads per thread, so that a CTA
// lives for a couple of gather round trips and does not hold an SM the forward kernels of other contexts are waiting for.
constexpr int ALIGN_THREADS = 128, ALIGN_BAND = 8;

// Least-squares similarity from the five landmarks p (image pixels) to the template q, centred closed form:
// a = sum(p~ . q~) / sum |p~|^2, b = sum(p~x q~y - p~y q~x) / sum |p~|^2, M = [[a, -b, tx], [b, a, ty]] (the minimiser
// Umeyama's SVD form finds).  Returns false (M = 0) when the landmarks coincide.
__device__ bool fit_similarity(const rf_face &f, float scale, const double *q, double M[6]) {
    double px[5], py[5];
    double pmx = 0.0, pmy = 0.0, qmx = 0.0, qmy = 0.0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        px[k] = (double)__fmul_rn(f.lx[k], scale);      // the map-back of k_merge_views
        py[k] = (double)__fmul_rn(f.ly[k], scale);
        pmx += px[k]; pmy += py[k]; qmx += q[2 * k]; qmy += q[2 * k + 1];
    }
    pmx /= 5.0; pmy /= 5.0; qmx /= 5.0; qmy /= 5.0;
    double den = 0.0, sxx = 0.0, sxy = 0.0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        const double ux = px[k] - pmx, uy = py[k] - pmy, vx = q[2 * k] - qmx, vy = q[2 * k + 1] - qmy;
        den += ux * ux + uy * uy;
        sxx += ux * vx + uy * vy;
        sxy += ux * vy - uy * vx;
    }
    if (den == 0.0) {
        for (int k = 0; k < 6; k++) M[k] = 0.0;
        return false;
    }
    const double a = sxx / den, b = sxy / den;
    M[0] = a; M[1] = -b; M[2] = qmx - a * pmx + b * pmy;
    M[3] = b; M[4] = a;  M[5] = qmy - b * pmx - a * pmy;
    return true;
}

// cv::invertAffineTransform (double)
__device__ void invert_affine(const double m[6], double im[6]) {
    double D = m[0] * m[4] - m[1] * m[3];
    D = D != 0.0 ? 1.0 / D : 0.0;
    const double a11 = m[4] * D, a22 = m[0] * D, a12 = -m[1] * D, a21 = -m[3] * D;
    im[0] = a11; im[1] = a12; im[2] = -a11 * m[2] - a12 * m[5];
    im[3] = a21; im[4] = a22; im[5] = -a21 * m[2] - a22 * m[5];
}

// One output pixel of cv::warpAffine INTER_LINEAR / BORDER_CONSTANT 0 on 8UC3: X, Y in 1/32 source pixel (X0 + adelta >> 5),
// integer weights 32 (32 - fx) (32 - fy) ... summing to 32768, taps outside the image contribute 0, (sum + 16384) >> 15.
__device__ __forceinline__ void tap(const AlignImageT<BgrRows> &im, int x, int y, int p[3]) {
    const uint8_t *q = im.src.p + (size_t)y * im.src.pitch + (size_t)x * 3;
    p[0] = q[0]; p[1] = q[1]; p[2] = q[2];
}
__device__ __forceinline__ void tap(const AlignImageT<YuvPlanes> &im, int x, int y, int p[3]) { yuv_pixel(im.src, x, y, p); }
// displayed pixel (x, y) of an oriented image: reflected, then transposed, as the letter-box reads it (preprocess.cu)
template <typename Img>
__device__ __forceinline__ void oriented_tap(const Img &im, int x, int y, int p[3]) {
    if (im.orient & LB_FLIP_X) x = im.w - 1 - x;
    if (im.orient & LB_FLIP_Y) y = im.h - 1 - y;
    if (im.orient & LB_TRANSPOSE) tap(im, y, x, p);
    else tap(im, x, y, p);
}

template <bool ORIENTED, typename Img>
__device__ __forceinline__ void sample(const Img &im, int X, int Y, int v[3]) {
    const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);   // saturate_cast<short>
    const int fx = X & 31, fy = Y & 31;
    const int wts[4] = {32 * (32 - fx) * (32 - fy), 32 * fx * (32 - fy), 32 * (32 - fx) * fy, 32 * fx * fy};
    int acc[3] = {16384, 16384, 16384};
#pragma unroll
    for (int t = 0; t < 4; t++) {
        const int tx = sx + (t & 1), ty = sy + (t >> 1);
        if ((unsigned)tx < (unsigned)im.w && (unsigned)ty < (unsigned)im.h) {
            int p[3];
            if (ORIENTED) oriented_tap(im, tx, ty, p);
            else tap(im, tx, ty, p);
            acc[0] += wts[t] * p[0]; acc[1] += wts[t] * p[1]; acc[2] += wts[t] * p[2];
        }
    }
    v[0] = acc[0] >> 15; v[1] = acc[1] >> 15; v[2] = acc[2] >> 15;
}

// A launch's chunk of the image table.  Only the oriented tables (f9) read `orient`: the other instantiations keep their code.
template <typename Src, bool O>
struct AlignTable {
    static constexpr bool kOriented = O;
    AlignImageT<Src> img[align_table_limit<Src>()];
};
static_assert(sizeof(AlignImageT<BgrRows>) == 32, "64 BGR images per launch rely on the 32-byte entry");
static_assert(sizeof(AlignArgs) + sizeof(AlignTable<BgrRows, false>) + 32 <= 4096 &&
              sizeof(AlignArgs) + sizeof(AlignTable<YuvPlanes, false>) + 32 <= 4096,
              "align launch exceeds the classic 4 KB kernel parameter space");

// Four consecutive pixels of one crop row (x4 .. x4 + 3, those < cw valid).  Vector stores where the address allows.
__device__ __forceinline__ void store_quad(const AlignArgs &a, unsigned char *crop, int y, int x4, const int v[4][3]) {
    const int cw = a.crop_w;
    const int nv = min(4, cw - x4);
    if (a.format == RF_CROP_BGR_U8) {
        unsigned char *d = crop + ((size_t)y * cw + x4) * 3;
        if (nv == 4 && ((uintptr_t)d & 3) == 0) {
            uint32_t *o = reinterpret_cast<uint32_t *>(d);
            o[0] = v[0][0] | (v[0][1] << 8) | (v[0][2] << 16) | ((uint32_t)v[1][0] << 24);
            o[1] = v[1][1] | (v[1][2] << 8) | (v[2][0] << 16) | ((uint32_t)v[2][1] << 24);
            o[2] = v[2][2] | (v[3][0] << 8) | (v[3][1] << 16) | ((uint32_t)v[3][2] << 24);
        } else {
            for (int k = 0; k < nv; k++)
                for (int c = 0; c < 3; c++) d[3 * k + c] = (unsigned char)v[k][c];
        }
        return;
    }
    const size_t plane = (size_t)a.crop_h * cw, off = (size_t)y * cw + x4;
#pragma unroll
    for (int c = 0; c < 3; c++) {                 // planes R, G, B = BGR channels 2, 1, 0
        float f[4];
#pragma unroll
        for (int k = 0; k < 4; k++) f[k] = __fmul_rn(__fsub_rn((float)v[k][2 - c], a.mean), a.inv_std);
        if (a.format == RF_CROP_RGB_F32) {
            float *d = reinterpret_cast<float *>(crop) + c * plane + off;
            if (nv == 4 && ((uintptr_t)d & 15) == 0) *reinterpret_cast<float4 *>(d) = make_float4(f[0], f[1], f[2], f[3]);
            else for (int k = 0; k < nv; k++) d[k] = f[k];
        } else {
            __half *d = reinterpret_cast<__half *>(crop) + c * plane + off;
            if (nv == 4 && ((uintptr_t)d & 7) == 0) {
                __half2 lo = __floats2half2_rn(f[0], f[1]), hi = __floats2half2_rn(f[2], f[3]);
                *reinterpret_cast<uint2 *>(d) = make_uint2(*reinterpret_cast<uint32_t *>(&lo), *reinterpret_cast<uint32_t *>(&hi));
            } else {
                for (int k = 0; k < nv; k++) d[k] = __float2half_rn(f[k]);
            }
        }
    }
}

// Every CTA first turns the kept counts of the n images into the crop ordinal of each image's first crop (a block scan of
// min(count_i, max_align)), then grid-strides over the row bands of the crops that exist -- the bands of a crop are
// consecutive work items -- so that free slots cost nothing however large max_align is.  Per item, thread 0 fits the
// transform in FP64, the CTA tabulates OpenCV's per-column (adelta, bdelta) and the band's per-row (X0, Y0) fixed-point
// terms in shared memory, and every pixel costs integer arithmetic only.
template <typename Table>
__global__ void __launch_bounds__(ALIGN_THREADS) k_align_faces(const AlignArgs a, const __grid_constant__ Table table, const rf_det *__restrict__ dets,
                                                             const int *__restrict__ counts, int max_faces) {
    extern __shared__ int s_first[];     // [n]: crop ordinal of image i's first crop
    __shared__ int s_ax[ALIGN_MAX_SIDE], s_bx[ALIGN_MAX_SIDE], s_x0[ALIGN_BAND], s_y0[ALIGN_BAND];
    __shared__ int s_wsum[ALIGN_THREADS / 32];
    __shared__ double s_im[6];
    __shared__ int s_zero;
    const int n = a.n, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    {
        // each thread a contiguous chunk of images; inclusive scan of the chunk sums over the block
        const int per = (n + ALIGN_THREADS - 1) / ALIGN_THREADS, lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
        int sum = 0;
        for (int i = lo; i < hi; i++) {
            const int k = min(min(counts[i], max_faces), a.max_align);
            s_first[i] = k;
            sum += k;
        }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_wsum[warp] = incl;
        __syncthreads();
        int run = incl - sum;
        for (int w = 0; w < warp; w++) run += s_wsum[w];
        for (int i = lo; i < hi; i++) {
            const int k = s_first[i];
            s_first[i] = run;
            run += k;
        }
    }
    int total = 0;
#pragma unroll
    for (int w = 0; w < ALIGN_THREADS / 32; w++) total += s_wsum[w];
    __syncthreads();
    const int cw = a.crop_w, ch = a.crop_h, qpr = (cw + 3) >> 2;
    const int bands = (ch + ALIGN_BAND - 1) / ALIGN_BAND, items = total * bands;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int c = item / bands, band = item - c * bands;
        int i = 0, top = n - 1;          // the last image whose first crop is <= c (images without crops share the next start)
        while (i < top) {
            const int mid = (i + top + 1) >> 1;
            if (s_first[mid] <= c) i = mid; else top = mid - 1;
        }
        const int j = c - s_first[i], slot = i * a.max_align + j;
        const auto im = table.img[i];
        if (threadIdx.x == 0) {
            double M[6], iM[6];
            s_zero = fit_similarity(dets[(size_t)i * max_faces + j].face, im.scale, a.tmpl, M) ? 0 : 1;
            invert_affine(M, iM);
            for (int k = 0; k < 6; k++) s_im[k] = iM[k];
            if (a.mats && band == 0)
                for (int k = 0; k < 6; k++) a.mats[(size_t)slot * 6 + k] = M[k];
        }
        __syncthreads();
        const double i0 = s_im[0], i1 = s_im[1], i2 = s_im[2], i3 = s_im[3], i4 = s_im[4], i5 = s_im[5];
        for (int x = threadIdx.x; x < cw; x += blockDim.x) {
            s_ax[x] = __double2int_rn(i0 * x * 1024.0);
            s_bx[x] = __double2int_rn(i3 * x * 1024.0);
        }
        const int ybase = band * ALIGN_BAND, rows = min(ALIGN_BAND, ch - ybase);
        if (threadIdx.x < rows) {
            const int y = ybase + threadIdx.x;
            s_x0[threadIdx.x] = __double2int_rn((i1 * y + i2) * 1024.0) + 16;
            s_y0[threadIdx.x] = __double2int_rn((i4 * y + i5) * 1024.0) + 16;
        }
        __syncthreads();
        const bool zero = s_zero != 0;
        unsigned char *crop = reinterpret_cast<unsigned char *>(a.crops) + (size_t)slot * a.crop_bytes;
        for (int qd = threadIdx.x; qd < rows * qpr; qd += blockDim.x) {
            const int r = qd / qpr, x4 = (qd - r * qpr) * 4;
            int v[4][3];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int x = x4 + k;
                if (x < cw && !zero) sample<Table::kOriented>(im, (s_x0[r] + s_ax[x]) >> 5, (s_y0[r] + s_bx[x]) >> 5, v[k]);
                else v[k][0] = v[k][1] = v[k][2] = 0;
            }
            store_quad(a, crop, ybase + r, x4, v);
        }
        __syncthreads();     // the tables of the next item overwrite these
    }
}

// Chunk i0 is its own launch over images [i0, i0 + m): the same kernel on offset records, counts, crops and matrices.  Two small
// CTAs per SM: the crops of a batch-8 step (about 40 faces x 14 bands) in one or two items per CTA, without taking more than a
// quarter of any SM's registers from the forward kernels of other contexts running alongside.
template <typename Table, typename Src>
cudaError_t launch_table(const AlignArgs &a, const AlignImageT<Src> *table, const PostBuffers &pb, int num_sms, cudaStream_t s) {
    constexpr int kMax = align_table_limit<Src>();
    for (int i0 = 0; i0 < a.n; i0 += kMax) {
        const int m = std::min(kMax, a.n - i0);
        AlignArgs c = a;
        c.n = m;
        c.crops = static_cast<unsigned char *>(a.crops) + (size_t)i0 * a.max_align * a.crop_bytes;
        if (a.mats) c.mats = a.mats + (size_t)i0 * a.max_align * 6;
        Table t{};
        for (int i = 0; i < m; i++) t.img[i] = table[i0 + i];
        k_align_faces<<<2 * num_sms, ALIGN_THREADS, sizeof(int) * m, s>>>(c, t, pb.out_dets + (size_t)i0 * pb.max_faces, pb.out_counts + i0,
                                                                        pb.max_faces);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace

template <typename Src>
cudaError_t launch_align_faces(const AlignArgs &a, const AlignImageT<Src> *table, const PostBuffers &pb, int num_sms, cudaStream_t s, bool oriented) {
    if (a.n <= 0 || a.max_align <= 0) return cudaSuccess;
    return oriented ? launch_table<AlignTable<Src, true>>(a, table, pb, num_sms, s) : launch_table<AlignTable<Src, false>>(a, table, pb, num_sms, s);
}

template cudaError_t launch_align_faces<BgrRows>(const AlignArgs &, const AlignImageT<BgrRows> *, const PostBuffers &, int, cudaStream_t, bool);
template cudaError_t launch_align_faces<YuvPlanes>(const AlignArgs &, const AlignImageT<YuvPlanes> *, const PostBuffers &, int, cudaStream_t, bool);

}  // namespace rf

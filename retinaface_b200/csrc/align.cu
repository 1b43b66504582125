// align.cu -- see align.cuh.  Compiled with -fmad=false: OpenCV evaluates iM01 * y + iM02 (and the closed-form sums here
// mirror oracle/align.py) as a separate multiply and add, and a contracted FMA can move a coordinate across a 1/1024
// rounding boundary.
#include "warp.cuh"

namespace rf {

size_t align_crop_bytes(int crop_w, int crop_h, int format) {
    const size_t px = (size_t)crop_w * crop_h * 3;
    return format == RF_CROP_RGB_F32 ? px * 4 : format == RF_CROP_RGB_F16 ? px * 2 : px;
}

namespace {

// A work item is one band of ALIGN_BAND crop rows of one (image, face) slot: about two pixel quads per thread, so that a CTA
// lives for a couple of gather round trips and does not hold an SM the forward kernels of other contexts are waiting for.
constexpr int ALIGN_THREADS = 128, ALIGN_BAND = 8;

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

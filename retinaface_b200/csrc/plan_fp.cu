// plan_fp.cu -- the FP32 / FP16 layer plan of the engine: which kernel runs which layers of the reference's graph
// (model/mnet-deconv-0517.prototxt), with which fused epilogues, on which lane of the forward graph.
#include "engine_internal.cuh"
#include "kernels_simt.cuh"
#include "stem_tc.cuh"
#include "tc_conv.cuh"
#include "tc_dwpw2d.cuh"

namespace rf_eng {

#define CK_L(...) CK(launch_k(__VA_ARGS__))

// GEMM weight matrix [K = (tap, cin)][N] from conv weights [cout][cin][k][k]; several convs that
// share an input are concatenated along N (det_conv1 + context_conv1, context_conv2 + conv3_1).
std::vector<float> pack_gemm(const std::vector<const FoldedConv *> &cs, std::vector<float> &bias) {
    const int cin = cs[0]->cin, k = cs[0]->k;
    int N = 0;
    for (auto c : cs) N += c->cout;
    std::vector<float> w((size_t)k * k * cin * N);
    bias.assign(N, 0.f);
    int n0 = 0;
    for (auto c : cs) {
        for (int o = 0; o < c->cout; o++) {
            bias[n0 + o] = c->b[o];
            for (int ci = 0; ci < cin; ci++)
                for (int t = 0; t < k * k; t++)
                    w[((size_t)t * cin + ci) * N + n0 + o] = c->w[((size_t)o * cin + ci) * k * k + t];
        }
        n0 += c->cout;
    }
    return w;
}

template <typename T>
void launch_gemm(const T *in, int ldin, int cin, const float *wk, const float *bias, int N, int ks, OutSplit<T> outs,
                 int n, int H, int W, cudaStream_t s) {
    long M = (long)n * H * W;
    int bn = (N % 64 == 0) ? 64 : (N % 32 == 0 ? 32 : 16);
    dim3 grid((unsigned)((M + 63) / 64), (N + bn - 1) / bn);
#define RF_GEMM(BN_, KS_) CK_L(k_conv_gemm<T, BN_, KS_>, grid, dim3(256), 0, s, in, ldin, cin, wk, bias, N, outs, n, H, W)
    if (ks == 1) { if (bn == 64) RF_GEMM(64, 1); else if (bn == 32) RF_GEMM(32, 1); else RF_GEMM(16, 1); }
    else { if (bn == 64) RF_GEMM(64, 3); else if (bn == 32) RF_GEMM(32, 3); else RF_GEMM(16, 3); }
#undef RF_GEMM
}

// ---- tensor-core path helpers ----------------------------------------------------------------
// B operand image [K/8][n][8] halfs (K-major no-swizzle, LBO = n*16 B), K ordered (tap, cin) and
// zero-padded to a multiple of 16; convs sharing an input are concatenated along N; `nsplit` slices
// of N each get their own image (slice s at s * Kpad * (N/nsplit)).
std::vector<__half> pack_tc_weights(const std::vector<const FoldedConv *> &cs, std::vector<float> &bias, int &Kpad, int nsplit) {
    const int cin = cs[0]->cin, k = cs[0]->k;
    int N = 0;
    for (auto c : cs) N += c->cout;
    const int K = k * k * cin;
    Kpad = (K + 15) / 16 * 16;
    const int Ns = N / nsplit;
    std::vector<__half> img((size_t)Kpad * N, __float2half(0.f));
    bias.assign(N, 0.f);
    int n0 = 0;
    for (auto c : cs) {
        for (int o = 0; o < c->cout; o++) {
            const int n = n0 + o, sl = n / Ns, nl = n % Ns;
            bias[n] = c->b[o];
            for (int ci = 0; ci < cin; ci++)
                for (int t = 0; t < k * k; t++) {
                    const int kk = t * cin + ci;
                    img[(size_t)sl * Kpad * Ns + ((size_t)(kk / 8) * Ns + nl) * 8 + (kk % 8)] =
                        __float2half(c->w[((size_t)o * cin + ci) * k * k + t]);
                }
        }
        n0 += c->cout;
    }
    return img;
}

void launch_tc_conv(const TcConvArgs &a_in, cudaStream_t s) {
    TcConvArgs a = a_in;
    a.mul_Wp = fast_div_mul((uint32_t)a.Wp); a.mul_Hp = fast_div_mul((uint32_t)a.Hp); a.mul_H = fast_div_mul((uint32_t)a.H);
    const long P = (long)a.nimg * a.Hp * a.Wp;
    const unsigned grid = (unsigned)((P + 127) / 128);
    const size_t smem = tc_conv_smem_bytes(a);
    switch (tc_n_bucket(a.N)) {
        case 32: if (a.up) CK_L(k_tc_conv_staged<32, true>, dim3(grid), dim3(TC_THREADS), smem, s, a); else CK_L(k_tc_conv_staged<32, false>, dim3(grid), dim3(TC_THREADS), smem, s, a); break;
        case 64: if (a.up) CK_L(k_tc_conv_staged<64, true>, dim3(grid), dim3(TC_THREADS), smem, s, a); else CK_L(k_tc_conv_staged<64, false>, dim3(grid), dim3(TC_THREADS), smem, s, a); break;
        case 128: if (a.up) CK_L(k_tc_conv_staged<128, true>, dim3(grid), dim3(TC_THREADS), smem, s, a); else CK_L(k_tc_conv_staged<128, false>, dim3(grid), dim3(TC_THREADS), smem, s, a); break;
        default: if (a.up) CK_L(k_tc_conv_staged<256, true>, dim3(grid), dim3(TC_THREADS), smem, s, a); else CK_L(k_tc_conv_staged<256, false>, dim3(grid), dim3(TC_THREADS), smem, s, a); break;
    }
}
void launch_tc_dwpw(const TcDwArgs &a_in, int nsplit, cudaStream_t s) {
    TcDwArgs a = a_in;
    a.mul_Wp = fast_div_mul((uint32_t)a.Wp); a.mul_Hp = fast_div_mul((uint32_t)a.Hp);
    a.mul_OW = fast_div_mul((uint32_t)a.OW); a.mul_OH = fast_div_mul((uint32_t)a.OH);
    const long M = (long)a.nimg * a.OH * a.OW;
    dim3 grid((unsigned)((M + a.rows - 1) / a.rows), nsplit);
    const size_t smem = tc_dw_smem_bytes(a);
    switch (tc_n_bucket(a.N)) {
        case 32: CK_L(k_tc_dwpw_staged<32>, grid, dim3(TC_THREADS), smem, s, a); break;
        case 64: CK_L(k_tc_dwpw_staged<64>, grid, dim3(TC_THREADS), smem, s, a); break;
        case 128: CK_L(k_tc_dwpw_staged<128>, grid, dim3(TC_THREADS), smem, s, a); break;
        default: CK_L(k_tc_dwpw_staged<256>, grid, dim3(TC_THREADS), smem, s, a); break;
    }
}
// the k_tc_dwpw_2d instantiation of a layer with N output channels
static void (*dw2d_kernel(int N))(TcDw2dArgs) {
    switch (tc_n_bucket(N)) {
        case 32: return k_tc_dwpw_2d<32>;
        case 64: return k_tc_dwpw_2d<64>;
        case 128: return k_tc_dwpw_2d<128>;
        default: return k_tc_dwpw_2d<256>;
    }
}
// persistent: at most `resident` CTAs (resident_ctas of this layer's instantiation and shared memory), each over a run of tiles
void launch_tc_dwpw_2d(TcDw2dArgs a, int resident, cudaStream_t s) {
    const PersistentGrid pg = persistent_grid(a.tiles_x * a.tiles_y * a.nimg, resident);
    a.run = pg.run;
    CK_L(dw2d_kernel(a.N), dim3((unsigned)pg.grid), dim3(TC_THREADS), tc_dw2d_smem_bytes(a), s, a);
}

// CTAs of `kern` the whole device holds at once with `threads` threads and `smem` bytes of dynamic shared memory: the grid of
// the persistent kernels.  Queried once, when the plan is built for launches; a plan that is only described launches nothing.
int resident_ctas(rf_handle h, const void *kern, int threads, size_t smem) {
    if (!h->on_device) return h->num_sms;
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    if (per_sm < 1) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("a kernel with %zu bytes of dynamic shared memory does not fit an SM", smem)};
    return per_sm * h->num_sms;
}

cudaError_t tc_init() {
    cudaError_t e;
#define RF_TC_ATTR(K_) if ((e = cudaFuncSetAttribute(K_, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT))) return e
    RF_TC_ATTR((k_tc_conv_staged<32, false>)); RF_TC_ATTR((k_tc_conv_staged<64, false>)); RF_TC_ATTR((k_tc_conv_staged<128, false>)); RF_TC_ATTR((k_tc_conv_staged<256, false>));
    RF_TC_ATTR((k_tc_conv_staged<32, true>)); RF_TC_ATTR((k_tc_conv_staged<64, true>)); RF_TC_ATTR((k_tc_conv_staged<128, true>)); RF_TC_ATTR((k_tc_conv_staged<256, true>));
    RF_TC_ATTR(k_tc_dwpw_staged<32>); RF_TC_ATTR(k_tc_dwpw_staged<64>); RF_TC_ATTR(k_tc_dwpw_staged<128>); RF_TC_ATTR(k_tc_dwpw_staged<256>);
    RF_TC_ATTR(k_tc_dwpw_2d<32>); RF_TC_ATTR(k_tc_dwpw_2d<64>); RF_TC_ATTR(k_tc_dwpw_2d<128>); RF_TC_ATTR(k_tc_dwpw_2d<256>);
#undef RF_TC_ATTR
    return cudaSuccess;
}

// Tile geometry of one fused depthwise+pointwise layer: rows per CTA, N slices and the exact upper
// bound of the staged range, so that everything fits in shared memory.
DwGeom dw_geometry(int C, int N, int IH, int IW, int S) {
    const int OH = IH / S, OW = IW / S, Wp = IW + 2, Hp = IH + 1, Kpad = (C + 15) / 16 * 16;
    auto centre = [&](long m) { long ox = m % OW, oy = (m / OW) % OH, b = m / ((long)OW * OH); return (b * Hp + oy * S) * Wp + ox * S + 1; };
    for (int rows : {128, 64}) {
        if (rows == 128 && OH * OW <= 28 * 28) continue;   // small maps: more, smaller CTAs (latency bound)
        for (int nsplit : {1, 2, 4}) {
            if ((N / nsplit) % 16) continue;
            // tile starts shift against image boundaries with period lcm(rows, OH*OW): scan one full period
            // (+1 image) so that every alignment, including tiles straddling two images, is covered
            long g = rows, t = (long)OH * OW;
            while (t) { long u = g % t; g = t; t = u; }
            const long M = ((long)rows / g + 1) * OH * OW;
            int R = 0;
            for (long m0 = 0; m0 < M; m0 += rows) {
                long ml = std::min(m0 + rows, M) - 1;
                R = std::max(R, (int)(centre(ml) - centre(m0) + 2 * (Wp + 1) + 1));
            }
            R |= 1;
            TcDwArgs a{};
            a.C = C; a.Rmax = R; a.Kpad = Kpad; a.N = N / nsplit; a.rows = rows;
            if (R <= TC_MAX_R && tc_dw_smem_bytes(a) <= (size_t)TC_SMEM_LIMIT) return {rows, nsplit, R};
        }
    }
    return {0, 0, 0};
}

// Constants of the tensor-core stem (stem_tc.cuh) as one blob: conv0's folded FP32 weights as two FP16 pieces (hi + lo), the
// pointwise B image, then the FP32 constants.  w0: [27][8] (k = (tap*3 + c_bgr), out channel), wd: [9][8], wp: [8][16].
std::vector<__half> make_stem_blob(const std::vector<float> &w0, const std::vector<float> &b0, const std::vector<float> &wd,
                                          const std::vector<float> &bd, const std::vector<float> &wp, const std::vector<float> &bp) {
    std::vector<__half> b0img(2 * 4 * 16 * 8, __float2half(0.f)), b1img(2 * 16 * 8, __float2half(0.f));
    for (int k = 0; k < 27; k++)
        for (int o = 0; o < 8; o++) {
            const float wv = w0[k * 8 + o];
            const __half hi = __float2half(wv);
            b0img[((k / 8) * 16 + o) * 8 + (k % 8)] = hi;                                            // w = hi + lo
            b0img[((4 + k / 8) * 16 + o) * 8 + (k % 8)] = __float2half(wv - __half2float(hi));
        }
    for (int c = 0; c < 8; c++)
        for (int o = 0; o < 16; o++) b1img[(0 * 16 + o) * 8 + c] = __float2half(wp[c * 16 + o]);
    std::vector<__half> blob(STEM_CONST_BYTES / 2, __float2half(0.f));
    memcpy(blob.data(), b0img.data(), STEM_B0_BYTES);
    memcpy(reinterpret_cast<unsigned char *>(blob.data()) + STEM_B0_BYTES, b1img.data(), STEM_B1_BYTES);
    std::vector<float> fl;
    fl.insert(fl.end(), b0.begin(), b0.begin() + 8);
    fl.insert(fl.end(), wd.begin(), wd.begin() + 72);
    fl.insert(fl.end(), bd.begin(), bd.begin() + 8);
    fl.insert(fl.end(), bp.begin(), bp.begin() + 16);
    fl.insert(fl.end(), wp.begin(), wp.begin() + 128);
    memcpy(reinterpret_cast<unsigned char *>(blob.data()) + STEM_B0_BYTES + STEM_B1_BYTES, fl.data(), STEM_F_FLOATS * 4);
    return blob;
}


// ---- exported step creators (FP16 tensor-core engine): used by build_plan<__half> and by plan_tile.cu -----------------------
// depthwise i + pointwise i+1 as one round-1 kernel (k_tc_dwpw_staged / k_tc_dwpw_2d); returns the output tensor id
int plan_pair_legacy(Builder &B, int i, int tin, int ih, int iw) {
    rf_handle h = B.h;
    const Model &m = h->model;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    const FoldedConv &dw = m.conv("mobilenet0_conv" + std::to_string(i) + "_fwd");
    const FoldedConv &pw = m.conv("mobilenet0_conv" + std::to_string(i + 1) + "_fwd");
    const int C = dw.cout, S = dw.stride;
    std::vector<float> wd(9 * C);
    for (int c = 0; c < C; c++)
        for (int t = 0; t < 9; t++) wd[t * C + c] = dw.w[(size_t)c * 9 + t];
    size_t owd = B.add_weights(wd), obd = B.add_weights(dw.b);
    const int oh = ih / S, ow_ = iw / S;
    const int N = pw.cout;
    const DwGeom geo = dw_geometry(C, N, ih, iw, S);
    if (geo.rows == 0) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("layer mobilenet0_conv%d (%dx%d, %d channels) does not fit shared memory", i, iw, ih, C)};
    std::vector<float> bias;
    int Kpad = 0;
    std::vector<__half> img = pack_tc_weights({&pw}, bias, Kpad, geo.nsplit);
    size_t oimg = B.add_weights_h(img), obp = B.add_weights(bias);
    int tpw = B.tensor("mobilenet0_relu" + std::to_string(i + 1) + "_fwd", oh, ow_, N);
    Step s;
    s.name = fmt("tc_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
    s.in = {tin}; s.out = {tpw};
    s.flops_per_img = 2.0 * oh * ow_ * C * 9 + 2.0 * oh * ow_ * C * N;
    s.bytes_per_img = ((double)ih * iw * C + (double)oh * ow_ * N) * es;
    // large maps (> 56x56 outputs; measured: no gain below): 2-D tiles (tc_dwpw2d.cuh) -- half the staged halo, no position
    // table, vertical reuse
    const bool tiles2d = oh * ow_ > 56 * 56 && C >= 16 && C <= 64 && geo.nsplit == 1 && !(h->cfg.flags & RF_FLAG_DW_1D);
    TcDw2dArgs g2{};            // 2-D tile geometry (independent of the batch)
    int resident = 0;
    if (tiles2d) {
        s.name = fmt("tc2d_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
        g2.C = C; g2.IH = ih; g2.IW = iw; g2.OH = oh; g2.OW = ow_; g2.S = S; g2.N = N;
        g2.TH = 8;
        const int t16 = (ow_ + 15) / 16, t14 = (ow_ + 13) / 14;
        g2.TW = t14 < t16 ? 14 : 16;
        tc_dw2d_finish(g2);
        resident = resident_ctas(h, (const void *)dw2d_kernel(N), TC_THREADS, tc_dw2d_smem_bytes(g2));
    }
    s.launch = [=](const Run &r) {
        if (tiles2d) {
            TcDw2dArgs a = g2;
            a.in = T_(r, tin); a.nimg = r.n;
            a.wimg = h->d_weights_h + oimg; a.bias = Wd(obp); a.dw_w = Wd(owd); a.dw_b = Wd(obd); a.out = T_(r, tpw);
            launch_tc_dwpw_2d(a, resident, r.stream);
            return;
        }
        TcDwArgs a{};
        a.in = T_(r, tin); a.C = C; a.nimg = r.n; a.IH = ih; a.IW = iw; a.OH = oh; a.OW = ow_; a.S = S;
        a.N = N / geo.nsplit; a.Ntotal = N; a.Kpad = Kpad; a.rows = geo.rows; a.Wp = iw + 2; a.Hp = ih + 1; a.Rmax = geo.Rmax;
        a.wimg = h->d_weights_h + oimg; a.bias = Wd(obp); a.dw_w = Wd(owd); a.dw_b = Wd(obd); a.out = T_(r, tpw);
        launch_tc_dwpw(a, geo.nsplit, r.stream);
    };
    B.step(std::move(s));
    return tpw;
}

// 1x1 / 3x3 convolution (branches sharing an input concatenated along N, outputs split over two destinations) as one
// round-1 kernel (k_tc_conv_staged); tup >= 0: FPN merge fused into the staging
void plan_conv_legacy(Builder &B, const std::string &sname, std::vector<const FoldedConv *> cs, int tin, int ih, int iw, int t0, int ld0,
                      int off0, int n0, int relu0, int t1, int ld1, int off1, int relu1, int lane, int tup, int up_which) {
    rf_handle h = B.h;
    const Model &m = h->model;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    std::vector<float> bias;
    int Kpad = 0;
    std::vector<__half> img = pack_tc_weights(cs, bias, Kpad);
    size_t oimg = B.add_weights_h(img), ob = B.add_weights(bias);
    const int N = (int)bias.size(), cin = cs[0]->cin, ks = cs[0]->k;
    size_t oup = tup >= 0 ? B.add_weights(m.up_w[up_which]) : 0;
    if (cin & (cin - 1)) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("convolution %s: %d input channels (the tensor-core kernels index by shifts: powers of two only)", sname.c_str(), cin)};
    TcConvArgs probe{};
    probe.Cin = cin; probe.taps = ks * ks; probe.N = N; probe.R = (ks == 3 ? 128 + 2 * (iw + 3) : 128) | 1;
    if (tup >= 0) { probe.up = reinterpret_cast<const __half *>(1); probe.Cmax = (((probe.R / (iw + 2) + 2) / 2 + 3) * (iw / 2)) | 1; }
    if (tc_conv_smem_bytes(probe) > (size_t)TC_SMEM_LIMIT || probe.R > TC_MAX_R)
        throw PlanFail{RF_ERR_UNSUPPORTED, fmt("convolution %s (%dx%d map) does not fit shared memory", sname.c_str(), iw, ih)};
    Step s;
    s.name = "tc_" + sname;
    s.lane = lane;
    s.in = {tin};
    if (tup >= 0) s.in.push_back(tup);
    s.out = {t0};
    if (t1 >= 0) s.out.push_back(t1);
    s.flops_per_img = 2.0 * ih * iw * cin * ks * ks * N + (tup >= 0 ? 2.0 * ih * iw * cin * 4 : 0.0);
    s.bytes_per_img = ((double)ih * iw * cin + (double)ih * iw * N + (tup >= 0 ? (double)(ih / 2) * (iw / 2) * cin : 0.0)) * es;
    s.launch = [=](const Run &r) {
        TcConvArgs a{};
        a.in = T_(r, tin); a.Cin = cin; a.nimg = r.n; a.H = ih; a.W = iw; a.taps = ks * ks; a.N = N;
        a.Wp = ks == 3 ? iw + 2 : iw; a.Hp = ks == 3 ? ih + 1 : ih;
        a.R = (ks == 3 ? 128 + 2 * (iw + 3) : 128) | 1;
        a.wimg = h->d_weights_h + oimg; a.bias = Wd(ob);
        a.out = TcOut{T_(r, t0) + off0, ld0, n0, relu0, t1 >= 0 ? T_(r, t1) + off1 : nullptr, ld1, relu1};
        if (tup >= 0) { a.up = T_(r, tup); a.up_w = Wd(oup); a.Cmax = (((a.R / a.Wp + 2) / 2 + 3) * (iw / 2)) | 1; }
        launch_tc_conv(a, r.stream);
    };
    B.step(std::move(s));
}

// c1-level FPN merge as its own packed-FP16 kernel (k_fpn_merge_h2); returns the merged tensor id
int plan_fpn_merge_h2(Builder &B, const std::string &name, int tlat, int tup, int fh, int fw, int which) {
    rf_handle h = B.h;
    const Model &m = h->model;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    const double es = h->elem;
    std::vector<__half> uwh(16 * 64);
    for (int c = 0; c < 64; c++)
        for (int t = 0; t < 16; t++) uwh[t * 64 + c] = __float2half(m.up_w[which][c * 16 + t]);
    size_t ouw = B.add_weights_h(uwh);
    int plus = B.tensor(name, fh, fw, 64);
    Step s;
    s.name = "fpn_merge" + name + "_upsample+add_h2";
    s.in = {tlat, tup}; s.out = {plus};
    s.flops_per_img = 2.0 * fh * fw * 64 * 4;
    s.bytes_per_img = ((double)fh * fw * 64 * 2 + (double)(fh / 2) * (fw / 2) * 64) * es;
    s.launch = [=](const Run &r) {
        // 128 threads per block: a 56-pixel row is 448 (pixel, 8-channel) items = 3.5 blocks
        CK(launch_k(k_fpn_merge_h2, dim3((unsigned)((fw * 8 + 127) / 128), (unsigned)fh, (unsigned)r.n), dim3(128), 0, r.stream, (const __half *)T_(r, tlat), (const __half *)T_(r, tup),
                    (__half *)T_(r, plus), (const __half *)(h->d_weights_h + ouw), r.n, fh, fw, 64));
    };
    B.step(std::move(s));
    return plus;
}

// the three predictor 1x1 convs + softmax + decode of all levels (k_head_decode), then sort + NMS (k_nms)
template <typename T>
void plan_heads_and_nms(Builder &B, bool with_heads, bool with_nms) {
    rf_handle h = B.h;
    const Model &m = h->model;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<T *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    const int H = h->cfg.net_h, W = h->cfg.net_w;
    const int h32 = H / 32, w32 = W / 32, h16 = H / 16, w16 = W / 16, h8 = H / 8, w8 = W / 8;
    if (with_heads) {
        size_t hw_off[3], hb_off[3];
        const int strides[3] = {32, 16, 8};
        for (int l = 0; l < 3; l++) {
            std::string st = "_stride" + std::to_string(strides[l]);
            const FoldedConv *cs[3] = {&m.conv("face_rpn_cls_score" + st), &m.conv("face_rpn_bbox_pred" + st),
                                       &m.conv("face_rpn_landmark_pred" + st)};
            std::vector<float> w(32 * 64), b(32);
            int r = 0;
            for (auto c : cs)
                for (int o = 0; o < c->cout; o++, r++) {
                    b[r] = c->b[o];
                    for (int ci = 0; ci < 64; ci++) w[r * 64 + ci] = c->w[(size_t)o * 64 + ci];
                }
            hw_off[l] = B.add_weights(w);
            hb_off[l] = B.add_weights(b);
        }
        Step s;
        s.name = "heads_1x1+softmax+decode_all_levels";
        s.in = {h->feat_tensor[0], h->feat_tensor[1], h->feat_tensor[2]};
        double px = (double)h32 * w32 + (double)h16 * w16 + (double)h8 * w8;
        s.flops_per_img = 2.0 * px * 64 * 4;   // threshold-first: only cls logits are computed for every pixel
        s.bytes_per_img = px * 64 * es;
        int f0 = h->feat_tensor[0], f1 = h->feat_tensor[1], f2 = h->feat_tensor[2];
        size_t w0 = hw_off[0], w1 = hw_off[1], w2 = hw_off[2], b0 = hb_off[0], b1 = hb_off[1], b2 = hb_off[2];
        s.launch = [=](const Run &r) {
            const T *feat[3] = {T_(r, f0), T_(r, f1), T_(r, f2)};
            HeadWeights hws[3] = {{Wd(w0), Wd(b0), 1.f}, {Wd(w1), Wd(b1), 1.f}, {Wd(w2), Wd(b2), 1.f}};
            launch_head_decode<T>(feat, hws, h->lv, r.n, W, H, r.ctx.d_params, r.ctx.pb, r.blobs, r.stream, with_nms);
        };
        if (with_nms) s.name = "heads_1x1+softmax+decode+nms_all_levels";     // decode -> NMS in one launch (last block per image)
        h->head_step = (int)h->steps.size();
        B.step(std::move(s));
        if (with_nms) return;
    }
    if (with_nms) {
        Step s;
        s.name = "sort+nms";
        // the candidates come from the steps that produce the three SSH outputs (tile chains with fused predictors, possibly on
        // other lanes): naming those tensors as inputs makes the NMS wait for every one of them
        s.in = {h->feat_tensor[0], h->feat_tensor[1], h->feat_tensor[2]};
        s.flops_per_img = 0;
        s.bytes_per_img = 0;
        s.launch = [=](const Run &r) { launch_nms(r.n, r.ctx.d_params, r.ctx.pb, r.stream); };
        h->nms_step = (int)h->steps.size();
        B.step(std::move(s));
    }
}
template void plan_heads_and_nms<float>(Builder &, bool, bool);
template void plan_heads_and_nms<__half>(Builder &, bool, bool);

// fused tensor-core stem (conv0 + dw1 + pw2); returns the tensor id of mobilenet0_relu2_fwd
int plan_stem_tc(Builder &B) {
    rf_handle h = B.h;
    const Model &m = h->model;
    const int H = h->cfg.net_h, W = h->cfg.net_w;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    const int cur_h = H / 2, cur_w = W / 2;
    const FoldedConv &c0 = m.conv("mobilenet0_conv0_fwd"), &dw = m.conv("mobilenet0_conv1_fwd"), &pw = m.conv("mobilenet0_conv2_fwd");
    std::vector<float> w0(27 * 8), wd(72), wp(128);
    for (int o = 0; o < 8; o++)
        for (int cb = 0; cb < 3; cb++)
            for (int t = 0; t < 9; t++) w0[(t * 3 + cb) * 8 + o] = c0.w[((size_t)o * 3 + (2 - cb)) * 9 + t];
    for (int c = 0; c < 8; c++)
        for (int t = 0; t < 9; t++) wd[t * 8 + c] = dw.w[(size_t)c * 9 + t];
    for (int o = 0; o < 16; o++)
        for (int c = 0; c < 8; c++) wp[c * 16 + o] = pw.w[(size_t)o * 8 + c];
    size_t ow0 = B.add_weights(w0), ob0 = B.add_weights(c0.b), owd = B.add_weights(wd), obd = B.add_weights(dw.b),
           owp = B.add_weights(wp), obp = B.add_weights(pw.b);
    std::vector<__half> blob = make_stem_blob(w0, c0.b, wd, dw.b, wp, pw.b);
    size_t oblob = B.add_weights_h(blob);
    const bool simt_stem = (h->cfg.flags & (RF_FLAG_SIMT_STEM | RF_FLAG_NO_TENSORCORE)) != 0;
    int out = B.tensor("mobilenet0_relu2_fwd", cur_h, cur_w, 16);
    Step s;
    s.name = simt_stem ? "stem_conv0+dw1+pw2_u8_to_16ch" : "tc_stem_conv0+dw1+pw2_u8_to_16ch";
    s.out = {out};
    s.flops_per_img = 2.0 * cur_h * cur_w * (8 * 27 + 8 * 9 + 8 * 16);
    s.bytes_per_img = (double)H * W * 3 + (double)cur_h * cur_w * 16 * es;
    const int tiles = ((H / 2 + 15) / 16) * ((W / 2 + 15) / 16);
    const int resident = simt_stem ? 0 : resident_ctas(h, (const void *)k_stem_tc<__half>, 256, 0);
    s.launch = [=](const Run &r) {
        if (simt_stem) {
            StemWeights sw{Wd(ow0), Wd(ob0), Wd(owd), Wd(obd), Wd(owp), Wd(obp)};
            CK(launch_k(k_stem<__half>, dim3((unsigned)(tiles * r.n)), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, (__half *)T_(r, out), sw, r.n, H, W, 1.0f));
        } else {
            StemTcArgs a{reinterpret_cast<const unsigned char *>(h->d_weights_h + oblob)};
            const PersistentGrid pg = persistent_grid(tiles * r.n, resident);
            stem_tc_finish(a, H, W, pg.run);
            CK(launch_k(k_stem_tc<__half>, dim3((unsigned)pg.grid), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, (__half *)T_(r, out), a, r.n, H, W, 1.0f));
        }
    };
    B.step(std::move(s));
    return out;
}

template <typename T>
void build_plan(rf_handle h) {
    Builder B{h, h->cfg.net_h, h->cfg.net_w};
    const Model &m = h->model;
    const int H = h->cfg.net_h, W = h->cfg.net_w;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<T *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;

    // ---- stem ------------------------------------------------------------------------------------
    int first_pair = 1;
    int cur_h = H / 2, cur_w = W / 2, cur_c = 8;
    int cur = -1;
    bool stem_done = false;
    if constexpr (std::is_same<T, __half>::value) {
        if (h->use_tc) {
            // conv0 + dw1 + pw2 fused: the two dense layers on tensor cores (stem_tc.cuh), or all on CUDA cores
            // (kernels_simt.cuh k_stem) with RF_FLAG_SIMT_STEM
            cur = plan_stem_tc(B);
            cur_c = 16;
            first_pair = 3;
            stem_done = true;
        }
    }
    if (!stem_done) {
    cur = B.tensor("mobilenet0_relu0_fwd", cur_h, cur_w, 8);
    {
        const FoldedConv &c = m.conv("mobilenet0_conv0_fwd");
        std::vector<float> wk(27 * 8);
        for (int o = 0; o < 8; o++)
            for (int cb = 0; cb < 3; cb++)       // cb: BGR channel of the u8 image; network channel = 2 - cb (RGB)
                for (int t = 0; t < 9; t++) wk[(t * 3 + cb) * 8 + o] = c.w[((size_t)o * 3 + (2 - cb)) * 9 + t];
        size_t ow = B.add_weights(wk), ob = B.add_weights(c.b);
        int out = cur;
        Step s;
        s.name = "conv0_u8_3x3s2_bn_relu";
        s.out = {out};
        s.flops_per_img = 2.0 * cur_h * cur_w * 8 * 27;
        s.bytes_per_img = (double)H * W * 3 + (double)cur_h * cur_w * 8 * es;
        s.launch = [=](const Run &r) {
            long total = (long)r.n * (H / 2) * (W / 2);
            CK_L(k_conv0<T>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, T_(r, out), Wd(ow), Wd(ob), r.n, H, W);
        };
        B.step(std::move(s));
    }
    }
    // ---- 13 x (depthwise 3x3, pointwise 1x1) (prototxt:55-1192) -----------------------------
    int c1 = -1, c2 = -1, c3 = -1;
    for (int i = first_pair; i <= 26; i += 2) {
        const FoldedConv &dw = m.conv("mobilenet0_conv" + std::to_string(i) + "_fwd");
        const FoldedConv &pw = m.conv("mobilenet0_conv" + std::to_string(i + 1) + "_fwd");
        const int C = dw.cout, S = dw.stride;
        std::vector<float> wd(9 * C);
        for (int c = 0; c < C; c++)
            for (int t = 0; t < 9; t++) wd[t * C + c] = dw.w[(size_t)c * 9 + t];
        size_t owd = B.add_weights(wd), obd = B.add_weights(dw.b);
        const int ih = cur_h, iw = cur_w, oh = cur_h / S, ow_ = cur_w / S;
        int tin = cur;
        if constexpr (std::is_same<T, __half>::value) {
            if (h->use_tc) {
                // depthwise + pointwise fused: stencil from staged shared memory -> wgmma GEMM (tc_conv.cuh)
                cur = plan_pair_legacy(B, i, tin, ih, iw);
                cur_h = oh; cur_w = ow_; cur_c = pw.cout;
                if (i + 1 == 10) c1 = cur;
                if (i + 1 == 22) c2 = cur;
                if (i + 1 == 26) c3 = cur;
                continue;
            }
        }
        int tdw = B.tensor("mobilenet0_relu" + std::to_string(i) + "_fwd", oh, ow_, C);
        {
            Step s;
            s.name = fmt("dw%d_3x3s%d_c%d", i, S, C);
            s.in = {tin}; s.out = {tdw};
            s.flops_per_img = 2.0 * oh * ow_ * C * 9;
            s.bytes_per_img = ((double)ih * iw * C + (double)oh * ow_ * C) * es;
            s.launch = [=](const Run &r) {
                long total = (long)r.n * oh * ow_ * (C / 8);
                unsigned g = (unsigned)((total + 255) / 256);
                if (S == 1) CK_L(k_dw3x3<T, 1>, dim3(g), dim3(256), 0, r.stream, (const T *)T_(r, tin), T_(r, tdw), Wd(owd), Wd(obd), r.n, ih, iw, C);
                else CK_L(k_dw3x3<T, 2>, dim3(g), dim3(256), 0, r.stream, (const T *)T_(r, tin), T_(r, tdw), Wd(owd), Wd(obd), r.n, ih, iw, C);
            };
            B.step(std::move(s));
        }
        std::vector<float> bias;
        std::vector<float> wk = pack_gemm({&pw}, bias);
        size_t owp = B.add_weights(wk), obp = B.add_weights(bias);
        const int N = pw.cout;
        int tpw = B.tensor("mobilenet0_relu" + std::to_string(i + 1) + "_fwd", oh, ow_, N);
        {
            Step s;
            s.name = fmt("pw%d_1x1_%dto%d", i + 1, C, N);
            s.in = {tdw}; s.out = {tpw};
            s.flops_per_img = 2.0 * oh * ow_ * C * N;
            s.bytes_per_img = ((double)oh * ow_ * C + (double)oh * ow_ * N) * es;
            s.launch = [=](const Run &r) {
                OutSplit<T> o{T_(r, tpw), N, N, 1, nullptr, 0, 0};
                launch_gemm<T>(T_(r, tdw), C, C, Wd(owp), Wd(obp), N, 1, o, r.n, oh, ow_, r.stream);
            };
            B.step(std::move(s));
        }
        cur = tpw; cur_h = oh; cur_w = ow_; cur_c = N;
        if (i + 1 == 10) c1 = cur;
        if (i + 1 == 22) c2 = cur;
        if (i + 1 == 26) c3 = cur;
    }
    (void)cur_c;

    // ---- FPN + SSH (prototxt:1199-2302) -----------------------------------------------------
    auto conv_step = [&](const std::string &sname, std::vector<const FoldedConv *> cs, int tin, int ih, int iw,
                         int t0, int ld0, int off0, int n0, int relu0, int t1, int ld1, int off1, int relu1, int lane = 0,
                         int tup = -1, int up_which = 0) {
        if constexpr (std::is_same<T, __half>::value) {
            if (h->use_tc) {
                plan_conv_legacy(B, sname, cs, tin, ih, iw, t0, ld0, off0, n0, relu0, t1, ld1, off1, relu1, lane, tup, up_which);
                return;
            }
        }
        std::vector<float> bias;
        std::vector<float> wk = pack_gemm(cs, bias);
        size_t ow = B.add_weights(wk), ob = B.add_weights(bias);
        const int N = (int)bias.size(), cin = cs[0]->cin, ks = cs[0]->k;
        const int ldin = h->tensors[tin].c;
        Step s;
        s.name = sname;
        s.lane = lane;
        s.in = {tin};
        s.out = {t0};
        if (t1 >= 0) s.out.push_back(t1);
        s.flops_per_img = 2.0 * ih * iw * cin * ks * ks * N;
        s.bytes_per_img = ((double)ih * iw * cin + (double)ih * iw * N) * es;
        s.launch = [=](const Run &r) {
            OutSplit<T> o{T_(r, t0) + off0, ld0, n0, relu0, t1 >= 0 ? T_(r, t1) + off1 : nullptr, ld1, relu1};
            launch_gemm<T>(T_(r, tin), ldin, cin, Wd(ow), Wd(ob), N, ks, o, r.n, ih, iw, r.stream);
        };
        B.step(std::move(s));
    };
    auto ssh = [&](const std::string &lvname, int tin, int fh, int fw, int level, int lane) {
        const std::string p = "rf_" + lvname + "_det";
        int cat = B.tensor(p + "_concat_relu", fh, fw, 64);
        int ctx1 = B.tensor(p + "_context_conv1_relu", fh, fw, 16);
        int ctx31 = B.tensor(p + "_context_conv3_1_relu", fh, fw, 16);
        // det_conv1 (64->32, BN, ReLU after concat) + context_conv1 (64->16, BN, ReLU): one launch
        conv_step("ssh_" + lvname + "_conv1+ctx1_3x3_64to48", {&m.conv(p + "_conv1"), &m.conv(p + "_context_conv1")}, tin, fh,
                  fw, cat, 64, 0, 32, 1, ctx1, 16, 0, 1, lane);
        // context_conv2 (16->16 -> concat[32:48]) + context_conv3_1 (16->16, ReLU): one launch
        conv_step("ssh_" + lvname + "_ctx2+ctx3_1_3x3_16to32", {&m.conv(p + "_context_conv2"), &m.conv(p + "_context_conv3_1")},
                  ctx1, fh, fw, cat, 64, 32, 16, 1, ctx31, 16, 0, 1, lane);
        // context_conv3_2 (16->16 -> concat[48:64])
        conv_step("ssh_" + lvname + "_ctx3_2_3x3_16to16", {&m.conv(p + "_context_conv3_2")}, ctx31, fh, fw, cat, 64, 48, 16, 1,
                  -1, 0, 0, 0, lane);
        h->feat_tensor[level] = cat;
        // the concat tensor is written by three steps: make it live from the first of them
    };
    auto upadd = [&](const std::string &name, int tlat, int tup, int fh, int fw, int which) {
        size_t ow = B.add_weights(m.up_w[which]);
        int out = B.tensor(name, fh, fw, 64);
        Step s;
        s.name = "upsample_add" + name;
        s.in = {tlat, tup}; s.out = {out};
        s.flops_per_img = 2.0 * fh * fw * 64 * 4;
        s.bytes_per_img = ((double)fh * fw * 64 * 2 + (double)(fh / 2) * (fw / 2) * 64) * es;
        s.launch = [=](const Run &r) {
            long total = (long)r.n * fh * fw * 8;
            CK_L(k_upsample_add<T>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, r.stream, (const T *)T_(r, tlat), (const T *)T_(r, tup), T_(r, out), Wd(ow), r.n,
                     fh, fw, 64, fh / 2, fw / 2);
        };
        B.step(std::move(s));
        return out;
    };
    const int h32 = H / 32, w32 = W / 32, h16 = H / 16, w16 = W / 16, h8 = H / 8, w8 = W / 8;
    // Lanes: the forward graph is not a chain.  rf_c1_red_conv only needs C1 and rf_c2_lateral only C2,
    // so they run on side lanes while the backbone continues; each level's SSH head runs on a side lane
    // while the main lane walks the top-down path lat3 -> aggr2 -> aggr1 -> ssh_c1 (the critical path).
    // In TC mode the FPN merge (deconv-upsample + add) is fused into the aggr conv's staging.
    const bool lanes = h->use_tc;
    // A side-lane step may start as soon as its producer finishes, i.e. EARLIER than later main-lane steps:
    // the step list (which the arena's liveness analysis walks in order) must show it right after that
    // producer, otherwise its output could be placed on memory a concurrently running main step still uses.
    auto move_last_step_after_producer = [&](int tensor_id) {
        int pos = 0;
        for (int i = (int)h->steps.size() - 2; i >= 0 && !pos; i--)
            for (int t : h->steps[i].out) if (t == tensor_id) { pos = i + 1; break; }
        Step st = std::move(h->steps.back());
        h->steps.pop_back();
        h->steps.insert(h->steps.begin() + pos, std::move(st));
    };
    int lat3 = B.tensor("rf_c3_lateral_relu", h32, w32, 64);
    int lat2 = B.tensor("rf_c2_lateral_relu", h16, w16, 64);
    int lat1 = B.tensor("rf_c1_red_conv_relu", h8, w8, 64);
    conv_step("c1_red_1x1_64to64", {&m.conv("rf_c1_red_conv")}, c1, h8, w8, lat1, 64, 0, 64, 1, -1, 0, 0, 0, lanes ? 1 : 0);
    if (lanes) move_last_step_after_producer(c1);
    conv_step("c2_lateral_1x1_128to64", {&m.conv("rf_c2_lateral")}, c2, h16, w16, lat2, 64, 0, 64, 1, -1, 0, 0, 0, lanes ? 2 : 0);
    if (lanes) move_last_step_after_producer(c2);
    conv_step("c3_lateral_1x1_256to64", {&m.conv("rf_c3_lateral")}, c3, h32, w32, lat3, 64, 0, 64, 1, -1, 0, 0, 0);
    ssh("c3", lat3, h32, w32, 0, lanes ? 1 : 0);
    int aggr2 = B.tensor("rf_c2_aggr_relu", h16, w16, 64);
    if (h->use_tc) {
        conv_step("c2_upsample+add+aggr_3x3_64to64", {&m.conv("rf_c2_aggr")}, lat2, h16, w16, aggr2, 64, 0, 64, 1, -1, 0, 0, 0, 0, lat3, 0);
    } else {
        int plus0 = upadd("_plus0", lat2, lat3, h16, w16, 0);
        conv_step("c2_aggr_3x3_64to64", {&m.conv("rf_c2_aggr")}, plus0, h16, w16, aggr2, 64, 0, 64, 1, -1, 0, 0, 0);
    }
    ssh("c2", aggr2, h16, w16, 1, lanes ? 2 : 0);
    int aggr1 = B.tensor("rf_c1_aggr_relu", h8, w8, 64);
    // Fusing the merge into the aggr conv costs ~50 KB of shared memory: fine while the conv's tiles fit one
    // wave (c2 level), a loss once it forces a second wave (c1 level at batch 8: 207 tiles, 1 CTA/SM).
    const long c1_tiles = ((long)h->cfg.max_batch * (h8 + 1) * (w8 + 2) + 127) / 128;
    if (h->use_tc && c1_tiles <= h->num_sms) {
        conv_step("c1_upsample+add+aggr_3x3_64to64", {&m.conv("rf_c1_aggr")}, lat1, h8, w8, aggr1, 64, 0, 64, 1, -1, 0, 0, 0, 0, aggr2, 1);
    } else if (h->use_tc) {
        if constexpr (std::is_same<T, __half>::value) {
            int plus1 = plan_fpn_merge_h2(B, "_plus1", lat1, aggr2, h8, w8, 1);
            conv_step("c1_aggr_3x3_64to64", {&m.conv("rf_c1_aggr")}, plus1, h8, w8, aggr1, 64, 0, 64, 1, -1, 0, 0, 0);
        }
    } else {
        int plus1 = upadd("_plus1", lat1, aggr2, h8, w8, 1);
        conv_step("c1_aggr_3x3_64to64", {&m.conv("rf_c1_aggr")}, plus1, h8, w8, aggr1, 64, 0, 64, 1, -1, 0, 0, 0);
    }
    ssh("c1", aggr1, h8, w8, 2, 0);

    // ---- predictors + decode (fused) and NMS -------------------------------------------------
    plan_heads_and_nms<T>(B, true, true);
}

template void build_plan<float>(rf_handle h);
template void build_plan<__half>(rf_handle h);

}  // namespace rf_eng

// plan_fp.cu -- the SIMT layer plans (FP32, FP16 with RF_FLAG_NO_TENSORCORE) as operations of the network walk (plan_net.cu),
// and the FP16 tensor-core per-layer operations and launch helpers the FP16 plan (plan_tile.cu) falls back to.
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

// k_conv_gemm's N tile: the widest of 64, 32, 16 that divides N.  M tiles: 64 positions of the n x H x W map.
static int gemm_bn(int N) { return (N % 64 == 0) ? 64 : (N % 32 == 0 ? 32 : 16); }
static std::string gemm_geom(int N, int H, int W) { return fmt("BM=64 bn=%d H=%d W=%d", gemm_bn(N), H, W); }

template <typename T>
void launch_gemm(const T *in, int ldin, int cin, const float *wk, const float *bias, int N, int ks, OutSplit<T> outs,
                 int n, int H, int W, cudaStream_t s) {
    long M = (long)n * H * W;
    int bn = gemm_bn(N);
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
    a.stages = std::min(a.stages, a.run + 1);       // a run of one tile has no use for a third window's shared memory
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

// Constants of the tensor-core stem (stem_tc.cuh) as one blob: conv0's folded FP32 weights as two FP16 pieces (hi + lo), the
// pointwise B image, then the FP32 constants.  w0: [27][8] (k = (tap*3 + c_bgr), out channel), wd: [9][8], wp: [8][16].
static std::vector<__half> make_stem_blob(const StemPack &p, const std::vector<float> &b0, const std::vector<float> &bd, const std::vector<float> &bp) {
    std::vector<__half> b0img(2 * 4 * 16 * 8, __float2half(0.f)), b1img(2 * 16 * 8, __float2half(0.f));
    for (int k = 0; k < 27; k++)
        for (int o = 0; o < 8; o++) {
            const float wv = p.w0[k * 8 + o];
            const __half hi = __float2half(wv);
            b0img[((k / 8) * 16 + o) * 8 + (k % 8)] = hi;                                            // w = hi + lo
            b0img[((4 + k / 8) * 16 + o) * 8 + (k % 8)] = __float2half(wv - __half2float(hi));
        }
    for (int c = 0; c < 8; c++)
        for (int o = 0; o < 16; o++) b1img[(0 * 16 + o) * 8 + c] = __float2half(p.wp[c * 16 + o]);
    std::vector<__half> blob(STEM_CONST_BYTES / 2, __float2half(0.f));
    memcpy(blob.data(), b0img.data(), STEM_B0_BYTES);
    memcpy(reinterpret_cast<unsigned char *>(blob.data()) + STEM_B0_BYTES, b1img.data(), STEM_B1_BYTES);
    std::vector<float> fl;
    fl.insert(fl.end(), b0.begin(), b0.begin() + 8);
    fl.insert(fl.end(), p.wd.begin(), p.wd.begin() + 72);
    fl.insert(fl.end(), bd.begin(), bd.begin() + 8);
    fl.insert(fl.end(), bp.begin(), bp.begin() + 16);
    fl.insert(fl.end(), p.wp.begin(), p.wp.begin() + 128);
    memcpy(reinterpret_cast<unsigned char *>(blob.data()) + STEM_B0_BYTES + STEM_B1_BYTES, fl.data(), STEM_F_FLOATS * 4);
    return blob;
}

// ---- FP16 tensor-core operations (per layer): the FP16 plan where no tile chain runs ---------------------------------------
// depthwise i + pointwise i+1 as one kernel (k_tc_dwpw_staged / k_tc_dwpw_2d); returns the output tensor id
int plan_pair_tc(Builder &B, const PairNode &p, int tin) {
    rf_handle h = B.h;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    const FoldedConv &dw = *p.dw, &pw = *p.pw;
    const int i = p.i, ih = p.h, iw = p.w, C = dw.cout, S = dw.stride;
    size_t owd = B.add_weights(pack_dw(dw)), obd = B.add_weights(dw.b);
    const int oh = ih / S, ow_ = iw / S;
    const int N = pw.cout;
    const DwGeom geo = dw_geometry(C, N, ih, iw, S, [C](int rows, int Ns, int R) {
        TcDwArgs a{};
        a.C = C; a.Rmax = R; a.Kpad = (C + 15) / 16 * 16; a.N = Ns; a.rows = rows;
        return R <= TC_MAX_R && tc_dw_smem_bytes(a) <= (size_t)TC_SMEM_LIMIT;
    });
    if (geo.rows == 0) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("layer %s (%dx%d, %d channels) does not fit shared memory", dw.name.c_str(), iw, ih, C)};
    std::vector<float> bias;
    int Kpad = 0;
    std::vector<__half> img = pack_tc_weights({&pw}, bias, Kpad, geo.nsplit);
    size_t oimg = B.add_weights_h(img), obp = B.add_weights(bias);
    int tpw = B.tensor(p.out, oh, ow_, N);
    Step s;
    s.name = fmt("tc_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
    s.in = {tin}; s.out = {tpw};
    s.flops_per_img = 2.0 * oh * ow_ * C * 9 + 2.0 * oh * ow_ * C * N;
    s.bytes_per_img = ((double)ih * iw * C + (double)oh * ow_ * N) * es;
    int tw = dw2d_tile_w(h, C, oh, ow_, geo.nsplit);
    TcDw2dArgs g2{};            // 2-D tile geometry (independent of the batch)
    int resident = 0;
    if (tw) {
        g2.C = C; g2.IH = ih; g2.IW = iw; g2.OH = oh; g2.OW = ow_; g2.S = S; g2.N = N;
        g2.TH = 8; g2.TW = tw;
        tc_dw2d_finish(g2);
        // a ring of three staged windows where they fit, else two.  With several execution contexts, one CTA per SM, each
        // over a run of ceil(tiles / SMs): the SM's other slots stay free for the other contexts' kernels (DESIGN §3: faster
        // on the flagship than three CTAs per SM with runs a third as long, though slower as a kernel alone, so a
        // one-context handle keeps every slot)
        g2.stages = 3;
        if (tc_dw2d_smem_bytes(g2) > (size_t)TC_SMEM_LIMIT) g2.stages = 2;
        resident = resident_ctas(h, (const void *)dw2d_kernel(N), TC_THREADS, tc_dw2d_smem_bytes(g2));
        if (h->cfg.streams != 1) resident = std::min(resident, h->num_sms);
        if (!tc_dw2d_out_fits(g2)) tw = 0;      // the output tile does not fit a consumed window: the 1-D kernel
    }
    if (tw) {
        s.name = fmt("tc2d_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
        s.geom = fmt("TH=%d TW=%d OH=%d OW=%d tiles_x=%d tiles_y=%d stages=%d", g2.TH, g2.TW, oh, ow_, g2.tiles_x, g2.tiles_y, g2.stages);
    } else {
        s.geom = fmt("rows=%d nsplit=%d Rmax=%d OH=%d OW=%d", geo.rows, geo.nsplit, geo.Rmax, oh, ow_);
    }
    s.launch = [=](const Run &r) {
        if (tw) {
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

// 1x1 / 3x3 convolution as one kernel (k_tc_conv_staged), the FPN merge fused into its staging where c.up >= 0
void plan_conv_tc(Builder &B, const ConvNode &c) {
    rf_handle h = B.h;
    const Model &m = h->model;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    std::vector<float> bias;
    int Kpad = 0;
    std::vector<__half> img = pack_tc_weights(c.cs, bias, Kpad);
    size_t oimg = B.add_weights_h(img), ob = B.add_weights(bias);
    const int N = (int)bias.size(), cin = c.cs[0]->cin, ks = c.cs[0]->k, tin = c.in, ih = c.h, iw = c.w, tup = c.up;
    const ConvOut o0 = c.out[0], o1 = c.out[1];
    size_t oup = tup >= 0 ? B.add_weights(m.up_w[c.up_which]) : 0;
    if (cin & (cin - 1)) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("convolution %s: %d input channels (the tensor-core kernels index by shifts: powers of two only)", c.name.c_str(), cin)};
    TcConvArgs probe{};
    probe.Cin = cin; probe.taps = ks * ks; probe.N = N; probe.R = (ks == 3 ? 128 + 2 * (iw + 3) : 128) | 1;
    if (tup >= 0) { probe.up = reinterpret_cast<const __half *>(1); probe.Cmax = (((probe.R / (iw + 2) + 2) / 2 + 3) * (iw / 2)) | 1; }
    if (tc_conv_smem_bytes(probe) > (size_t)TC_SMEM_LIMIT || probe.R > TC_MAX_R)
        throw PlanFail{RF_ERR_UNSUPPORTED, fmt("convolution %s (%dx%d map) does not fit shared memory", c.name.c_str(), iw, ih)};
    Step s;
    s.name = "tc_" + c.name;
    s.lane = c.lane;
    s.in = {tin};
    if (tup >= 0) s.in.push_back(tup);
    s.out = {o0.t};
    if (o1.t >= 0) s.out.push_back(o1.t);
    s.flops_per_img = 2.0 * ih * iw * cin * ks * ks * N + (tup >= 0 ? 2.0 * ih * iw * cin * 4 : 0.0);
    s.bytes_per_img = ((double)ih * iw * cin + (double)ih * iw * N + (tup >= 0 ? (double)(ih / 2) * (iw / 2) * cin : 0.0)) * es;
    s.geom = fmt("NT=%d BM=128 H=%d W=%d Hp=%d Wp=%d merge=%s", tc_n_bucket(N), ih, iw, ks == 3 ? ih + 1 : ih, ks == 3 ? iw + 2 : iw,
                 tup >= 0 ? "fused" : "none");
    s.launch = [=](const Run &r) {
        TcConvArgs a{};
        a.in = T_(r, tin); a.Cin = cin; a.nimg = r.n; a.H = ih; a.W = iw; a.taps = ks * ks; a.N = N;
        a.Wp = ks == 3 ? iw + 2 : iw; a.Hp = ks == 3 ? ih + 1 : ih;
        a.R = (ks == 3 ? 128 + 2 * (iw + 3) : 128) | 1;
        a.wimg = h->d_weights_h + oimg; a.bias = Wd(ob);
        a.out = TcOut{T_(r, o0.t) + o0.off, o0.ld, o0.n, o0.relu, o1.t >= 0 ? T_(r, o1.t) + o1.off : nullptr, o1.ld, o1.relu};
        if (tup >= 0) { a.up = T_(r, tup); a.up_w = Wd(oup); a.Cmax = (((a.R / a.Wp + 2) / 2 + 3) * (iw / 2)) | 1; }
        launch_tc_conv(a, r.stream);
    };
    B.step(std::move(s));
}

// FPN merge as its own packed-FP16 kernel (k_fpn_merge_h2); returns the merged tensor id
int plan_fpn_merge_h2(Builder &B, const MergeNode &mn) {
    rf_handle h = B.h;
    const Model &m = h->model;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<__half *>(r.ctx.arena + h->tensors[id].offset); };
    const double es = h->elem;
    const int tlat = mn.lat, tup = mn.up, fh = mn.h, fw = mn.w;
    std::vector<__half> uwh(16 * 64);
    for (int c = 0; c < 64; c++)
        for (int t = 0; t < 16; t++) uwh[t * 64 + c] = __float2half(m.up_w[mn.level - 1][c * 16 + t]);
    size_t ouw = B.add_weights_h(uwh);
    int plus = B.tensor(mn.sum, fh, fw, 64);
    Step s;
    s.name = "fpn_merge" + mn.sum + "_upsample+add_h2";
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

// The three predictor 1x1 convs of every level + softmax + decode, then sort + NMS by the last block of each image, in one
// launch (k_head_decode); feature level l is dequantised by scale[l].
template <typename T>
void plan_heads(Builder &B, const HeadsNode &n, const float scale[3], const char *prefix) {
    rf_handle h = B.h;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<T *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    const int H = h->cfg.net_h, W = h->cfg.net_w;
    const int h32 = H / 32, w32 = W / 32, h16 = H / 16, w16 = W / 16, h8 = H / 8, w8 = W / 8;
    size_t hw_off[3], hb_off[3];
    for (int l = 0; l < 3; l++) {
        std::vector<float> w(32 * 64), b(32);
        int r = 0;
        for (auto c : n.pred[l])
            for (int o = 0; o < c->cout; o++, r++) {
                b[r] = c->b[o];
                for (int ci = 0; ci < 64; ci++) w[r * 64 + ci] = c->w[(size_t)o * 64 + ci];
            }
        hw_off[l] = B.add_weights(w);
        hb_off[l] = B.add_weights(b);
    }
    Step s;
    s.name = std::string(prefix) + "heads_1x1+softmax+decode+nms_all_levels";   // decode -> NMS in one launch (last block per image)
    s.in = {h->feat_tensor[0], h->feat_tensor[1], h->feat_tensor[2]};
    double px = (double)h32 * w32 + (double)h16 * w16 + (double)h8 * w8;
    s.flops_per_img = 2.0 * px * 64 * 4;   // threshold-first: only cls logits are computed for every pixel
    s.bytes_per_img = px * 64 * es;
    int f0 = h->feat_tensor[0], f1 = h->feat_tensor[1], f2 = h->feat_tensor[2];
    size_t w0 = hw_off[0], w1 = hw_off[1], w2 = hw_off[2], b0 = hb_off[0], b1 = hb_off[1], b2 = hb_off[2];
    float s0 = scale[0], s1 = scale[1], s2 = scale[2];
    s.launch = [=](const Run &r) {
        const T *feat[3] = {T_(r, f0), T_(r, f1), T_(r, f2)};
        HeadWeights hws[3] = {{Wd(w0), Wd(b0), s0}, {Wd(w1), Wd(b1), s1}, {Wd(w2), Wd(b2), s2}};
        CK(launch_head_decode<T>(feat, hws, h->lv, r.n, W, H, r.ctx.d_params, r.ctx.pb, r.blobs, r.stream, true));
    };
    B.step(std::move(s));
}
template void plan_heads<float>(Builder &, const HeadsNode &, const float[3], const char *);
template void plan_heads<__half>(Builder &, const HeadsNode &, const float[3], const char *);
template void plan_heads<int8_t>(Builder &, const HeadsNode &, const float[3], const char *);

// conv0 + dw1 + pw2 in one kernel: the two dense layers on tensor cores (stem_tc.cuh k_stem_tc), or all three on CUDA cores
// (kernels_simt.cuh k_stem) with RF_FLAG_SIMT_STEM; the output is scaled by out_scale (INT8: 1 / its table scale)
template <typename OutT>
int plan_stem_fused(Builder &B, const StemNode &n, const char *suffix, float out_scale) {
    rf_handle h = B.h;
    const int H = h->cfg.net_h, W = h->cfg.net_w;
    auto T_ = [h](const Run &r, int id) { return reinterpret_cast<OutT *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    const double es = h->elem;
    const int cur_h = H / 2, cur_w = W / 2;
    const StemPack p = pack_stem(n);
    size_t ow0 = B.add_weights(p.w0), ob0 = B.add_weights(n.conv0->b), owd = B.add_weights(p.wd), obd = B.add_weights(n.pair.dw->b),
           owp = B.add_weights(p.wp), obp = B.add_weights(n.pair.pw->b);
    size_t oblob = B.add_weights_h(make_stem_blob(p, n.conv0->b, n.pair.dw->b, n.pair.pw->b));
    const bool simt_stem = (h->cfg.flags & (RF_FLAG_SIMT_STEM | RF_FLAG_NO_TENSORCORE)) != 0;
    int out = B.tensor(n.pair.out, cur_h, cur_w, 16);
    Step s;
    s.name = std::string(simt_stem ? "" : "tc_") + "stem_conv0+dw1+pw2_u8_to_16ch" + suffix;
    s.out = {out};
    s.flops_per_img = 2.0 * cur_h * cur_w * (8 * 27 + 8 * 9 + 8 * 16);
    s.bytes_per_img = (double)H * W * 3 + (double)cur_h * cur_w * 16 * es;
    const int tiles = ((H / 2 + 15) / 16) * ((W / 2 + 15) / 16);
    s.geom = fmt("TH=16 TW=16 OH=%d OW=%d tiles_x=%d tiles_y=%d", cur_h, cur_w, (cur_w + 15) / 16, (cur_h + 15) / 16);
    const int resident = simt_stem ? 0 : resident_ctas(h, (const void *)k_stem_tc<OutT>, 256, 0);
    s.launch = [=](const Run &r) {
        if (simt_stem) {
            StemWeights sw{Wd(ow0), Wd(ob0), Wd(owd), Wd(obd), Wd(owp), Wd(obp)};
            CK_L(k_stem<OutT>, dim3((unsigned)(tiles * r.n)), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, T_(r, out), sw, r.n, H, W, out_scale);
        } else {
            StemTcArgs a{reinterpret_cast<const unsigned char *>(h->d_weights_h + oblob)};
            const PersistentGrid pg = persistent_grid(tiles * r.n, resident);
            stem_tc_finish(a, H, W, pg.run);
            CK_L(k_stem_tc<OutT>, dim3((unsigned)pg.grid), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, T_(r, out), a, r.n, H, W, out_scale);
        }
    };
    B.step(std::move(s));
    return out;
}
template int plan_stem_fused<__half>(Builder &, const StemNode &, const char *, float);
template int plan_stem_fused<int8_t>(Builder &, const StemNode &, const char *, float);

// ---- SIMT operations (FP32; FP16 with RF_FLAG_NO_TENSORCORE): every layer its own CUDA-core kernel, all steps on lane 0 -----
template <typename T>
struct SimtOps : PlanOps {
    using PlanOps::PlanOps;
    static T *t(rf_handle h, const Run &r, int id) { return reinterpret_cast<T *>(r.ctx.arena + h->tensors[id].offset); }

    int stem(const StemNode &n) override {
        rf_handle h = B.h;
        const int H = h->cfg.net_h, W = h->cfg.net_w, cur_h = H / 2, cur_w = W / 2;
        const int out = B.tensor(n.out0, cur_h, cur_w, 8);
        size_t ow = B.add_weights(pack_stem(n).w0), ob = B.add_weights(n.conv0->b);
        Step s;
        s.name = "conv0_u8_3x3s2_bn_relu";
        s.out = {out};
        s.flops_per_img = 2.0 * cur_h * cur_w * 8 * 27;
        s.bytes_per_img = (double)H * W * 3 + (double)cur_h * cur_w * 8 * h->elem;
        s.launch = [=](const Run &r) {
            long total = (long)r.n * (H / 2) * (W / 2);
            CK_L(k_conv0<T>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, t(h, r, out),
                 h->d_weights + ow, h->d_weights + ob, r.n, H, W);
        };
        B.step(std::move(s));
        return pair(n.pair, out);
    }

    int pair(const PairNode &p, int tin) override {
        rf_handle h = B.h;
        const FoldedConv &dw = *p.dw, &pw = *p.pw;
        const int C = dw.cout, S = dw.stride, N = pw.cout, i = p.i, ih = p.h, iw = p.w, oh = ih / S, ow_ = iw / S;
        const double es = h->elem;
        size_t owd = B.add_weights(pack_dw(dw)), obd = B.add_weights(dw.b);
        int tdw = B.tensor(p.mid, oh, ow_, C);
        Step s;
        s.name = fmt("dw%d_3x3s%d_c%d", i, S, C);
        s.in = {tin}; s.out = {tdw};
        s.flops_per_img = 2.0 * oh * ow_ * C * 9;
        s.bytes_per_img = ((double)ih * iw * C + (double)oh * ow_ * C) * es;
        s.launch = [=](const Run &r) {
            long total = (long)r.n * oh * ow_ * (C / 8);
            unsigned g = (unsigned)((total + 255) / 256);
            const float *w = h->d_weights + owd, *b = h->d_weights + obd;
            if (S == 1) CK_L(k_dw3x3<T, 1>, dim3(g), dim3(256), 0, r.stream, (const T *)t(h, r, tin), t(h, r, tdw), w, b, r.n, ih, iw, C);
            else CK_L(k_dw3x3<T, 2>, dim3(g), dim3(256), 0, r.stream, (const T *)t(h, r, tin), t(h, r, tdw), w, b, r.n, ih, iw, C);
        };
        B.step(std::move(s));
        std::vector<float> bias;
        std::vector<float> wk = pack_gemm({&pw}, bias);
        size_t owp = B.add_weights(wk), obp = B.add_weights(bias);
        int tpw = B.tensor(p.out, oh, ow_, N);
        Step s2;
        s2.name = fmt("pw%d_1x1_%dto%d", i + 1, C, N);
        s2.in = {tdw}; s2.out = {tpw};
        s2.flops_per_img = 2.0 * oh * ow_ * C * N;
        s2.bytes_per_img = ((double)oh * ow_ * C + (double)oh * ow_ * N) * es;
        s2.geom = gemm_geom(N, oh, ow_);
        s2.launch = [=](const Run &r) {
            OutSplit<T> o{t(h, r, tpw), N, N, 1, nullptr, 0, 0};
            launch_gemm<T>(t(h, r, tdw), C, C, h->d_weights + owp, h->d_weights + obp, N, 1, o, r.n, oh, ow_, r.stream);
        };
        B.step(std::move(s2));
        return tpw;
    }

    void conv(const ConvNode &c) override {      // c.lane is not used: one lane
        rf_handle h = B.h;
        std::vector<float> bias;
        std::vector<float> wk = pack_gemm(c.cs, bias);
        size_t ow = B.add_weights(wk), ob = B.add_weights(bias);
        const int N = (int)bias.size(), cin = c.cs[0]->cin, ks = c.cs[0]->k, tin = c.in, ih = c.h, iw = c.w;
        const int ldin = h->tensors[tin].c;
        const ConvOut o0 = c.out[0], o1 = c.out[1];
        Step s;
        s.name = c.name;
        s.in = {tin};
        s.out = {o0.t};
        if (o1.t >= 0) s.out.push_back(o1.t);
        s.flops_per_img = 2.0 * ih * iw * cin * ks * ks * N;
        s.bytes_per_img = ((double)ih * iw * cin + (double)ih * iw * N) * h->elem;
        s.geom = gemm_geom(N, ih, iw);
        s.launch = [=](const Run &r) {
            OutSplit<T> o{t(h, r, o0.t) + o0.off, o0.ld, o0.n, o0.relu, o1.t >= 0 ? t(h, r, o1.t) + o1.off : nullptr, o1.ld, o1.relu};
            launch_gemm<T>(t(h, r, tin), ldin, cin, h->d_weights + ow, h->d_weights + ob, N, ks, o, r.n, ih, iw, r.stream);
        };
        B.step(std::move(s));
    }

    int merge(const MergeNode &m) override {
        rf_handle h = B.h;
        size_t ow = B.add_weights(h->model.up_w[m.level - 1]);
        const int tlat = m.lat, tup = m.up, fh = m.h, fw = m.w;
        int out = B.tensor(m.sum, fh, fw, 64);
        Step s;
        s.name = "upsample_add" + m.sum;
        s.in = {tlat, tup}; s.out = {out};
        s.flops_per_img = 2.0 * fh * fw * 64 * 4;
        s.bytes_per_img = ((double)fh * fw * 64 * 2 + (double)(fh / 2) * (fw / 2) * 64) * h->elem;
        s.launch = [=](const Run &r) {
            long total = (long)r.n * fh * fw * 8;
            CK_L(k_upsample_add<T>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, r.stream, (const T *)t(h, r, tlat), (const T *)t(h, r, tup), t(h, r, out),
                 h->d_weights + ow, r.n, fh, fw, 64, fh / 2, fw / 2);
        };
        B.step(std::move(s));
        return out;
    }

    bool fuse_merge(const MergeNode &) override { return false; }

    void heads(const HeadsNode &n) override {
        const float one[3] = {1.f, 1.f, 1.f};
        plan_heads<T>(B, n, one, "");
    }
};

template <typename T>
void build_plan(rf_handle h) {
    SimtOps<T> ops(h);
    walk_network(ops);
}

template void build_plan<float>(rf_handle h);
template void build_plan<__half>(rf_handle h);

}  // namespace rf_eng

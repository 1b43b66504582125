// plan_i8.cu -- the INT8 layer plan of the engine (RF_PREC_INT8): the INT8 operations of the network walk (plan_net.cu).
#include "engine_internal.cuh"
#include "kernels_simt.cuh"
#include "tc_conv_i8.cuh"
#include "tc_dwpw2d_i8.cuh"

namespace rf_eng {

// =============================================================================================
// INT8 plan (RF_PREC_INT8): same graph, int8 activations with the calibration table's scales.
// The integer scheme is restated in oracle/mnet_int8.py (the checker); tensor scales are looked up by
// the Caffe top name each tensor carries.
// =============================================================================================
struct QWeights { std::vector<int8_t> img; std::vector<float> mult, bq; };

// cs: convs sharing an input, concatenated along N.  s_out[n]: quantisation scale of output channel n.
// Image: nsplit slices of N/nsplit channels, each [taps * groups][Ns][16] with `groups` 16-channel groups per tap
// (zero padded beyond cin).
QWeights pack_tc_weights_i8(const std::vector<const FoldedConv *> &cs, float s_in, const std::vector<float> &s_out, int groups, int nsplit) {
    const int cin = cs[0]->cin, k = cs[0]->k, taps = k * k;
    int N = 0;
    for (auto c : cs) N += c->cout;
    const int Ns = N / nsplit;
    QWeights q;
    q.img.assign((size_t)taps * groups * 16 * N, 0);
    q.mult.resize(N); q.bq.resize(N);
    int n0 = 0;
    for (auto c : cs) {
        const size_t per = (size_t)cin * taps;
        for (int o = 0; o < c->cout; o++) {
            const int n = n0 + o, sl = n / Ns, nl = n % Ns;
            float mx = 0.f;
            for (size_t i = 0; i < per; i++) mx = std::max(mx, std::fabs(c->w[o * per + i]));
            const float sw = mx > 0.f ? mx / 127.0f : 1.0f;
            q.mult[n] = (float)((double)s_in * (double)sw / (double)s_out[n]);
            q.bq[n] = (float)((double)c->b[o] / (double)s_out[n]);
            for (int ci = 0; ci < cin; ci++)
                for (int t = 0; t < taps; t++) {
                    double v = std::nearbyint((double)c->w[((size_t)o * cin + ci) * taps + t] / (double)sw);
                    v = std::max(-127.0, std::min(127.0, v));
                    const int g = t * groups + ci / 16;
                    q.img[(size_t)sl * taps * groups * 16 * Ns + ((size_t)g * Ns + nl) * 16 + (ci % 16)] = (int8_t)v;
                }
        }
        n0 += c->cout;
    }
    return q;
}

void launch_tc_conv_i8(const TcConvArgsI8 &a_in, cudaStream_t s) {
    TcConvArgsI8 a = a_in;
    a.mul_Wp = fast_div_mul((uint32_t)a.Wp); a.mul_Hp = fast_div_mul((uint32_t)a.Hp); a.mul_H = fast_div_mul((uint32_t)a.H);
    const long P = (long)a.nimg * a.Hp * a.Wp;
    const dim3 grid((unsigned)((P + 127) / 128));
    const size_t smem = tc_conv_i8_smem_bytes(a);
#define RF_I8C(NT_) if (a.up) CK(launch_k(k_tc_conv_staged_i8<NT_, true>, grid, dim3(TC_THREADS), smem, s, a)); else CK(launch_k(k_tc_conv_staged_i8<NT_, false>, grid, dim3(TC_THREADS), smem, s, a))
    switch (tc_n_bucket(a.N)) {
        case 32: RF_I8C(32); break;
        case 64: RF_I8C(64); break;
        case 128: RF_I8C(128); break;
        default: RF_I8C(256); break;
    }
#undef RF_I8C
}
void launch_tc_dwpw_2d_i8(const TcDw2dArgsI8 &a, cudaStream_t s) {
    const dim3 grid((unsigned)a.tiles_x, (unsigned)a.tiles_y, (unsigned)a.nimg);
    const size_t smem = tc_dw2d_i8_smem_bytes(a);
    switch (tc_n_bucket(a.N)) {
        case 32: CK(launch_k(k_tc_dwpw_2d_i8<32>, grid, dim3(TC_THREADS), smem, s, a)); break;
        case 64: CK(launch_k(k_tc_dwpw_2d_i8<64>, grid, dim3(TC_THREADS), smem, s, a)); break;
        case 128: CK(launch_k(k_tc_dwpw_2d_i8<128>, grid, dim3(TC_THREADS), smem, s, a)); break;
        default: CK(launch_k(k_tc_dwpw_2d_i8<256>, grid, dim3(TC_THREADS), smem, s, a)); break;
    }
}

void launch_tc_dwpw_i8(const TcDwArgsI8 &a_in, int nsplit, cudaStream_t s) {
    TcDwArgsI8 a = a_in;
    a.mul_Wp = fast_div_mul((uint32_t)a.Wp); a.mul_Hp = fast_div_mul((uint32_t)a.Hp);
    a.mul_OW = fast_div_mul((uint32_t)a.OW); a.mul_OH = fast_div_mul((uint32_t)a.OH);
    const long M = (long)a.nimg * a.OH * a.OW;
    const dim3 grid((unsigned)((M + a.rows - 1) / a.rows), nsplit);
    const size_t smem = tc_dw_i8_smem_bytes(a);
    switch (tc_n_bucket(a.N)) {
        case 32: if (a.C >= 64) CK(launch_k(k_tc_dwpw_staged_i8<32, true>, grid, dim3(TC_THREADS), smem, s, a)); else CK(launch_k(k_tc_dwpw_staged_i8<32, false>, grid, dim3(TC_THREADS), smem, s, a)); break;
        case 64: if (a.C >= 64) CK(launch_k(k_tc_dwpw_staged_i8<64, true>, grid, dim3(TC_THREADS), smem, s, a)); else CK(launch_k(k_tc_dwpw_staged_i8<64, false>, grid, dim3(TC_THREADS), smem, s, a)); break;
        case 128: if (a.C >= 64) CK(launch_k(k_tc_dwpw_staged_i8<128, true>, grid, dim3(TC_THREADS), smem, s, a)); else CK(launch_k(k_tc_dwpw_staged_i8<128, false>, grid, dim3(TC_THREADS), smem, s, a)); break;
        default: if (a.C >= 64) CK(launch_k(k_tc_dwpw_staged_i8<256, true>, grid, dim3(TC_THREADS), smem, s, a)); else CK(launch_k(k_tc_dwpw_staged_i8<256, false>, grid, dim3(TC_THREADS), smem, s, a)); break;
    }
}
cudaError_t tc_init_i8() {
    cudaError_t e;
#define RF_TC_ATTR(K_) if ((e = cudaFuncSetAttribute(K_, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT))) return e
    RF_TC_ATTR((k_tc_conv_staged_i8<32, false>)); RF_TC_ATTR((k_tc_conv_staged_i8<64, false>)); RF_TC_ATTR((k_tc_conv_staged_i8<128, false>)); RF_TC_ATTR((k_tc_conv_staged_i8<256, false>));
    RF_TC_ATTR((k_tc_conv_staged_i8<32, true>)); RF_TC_ATTR((k_tc_conv_staged_i8<64, true>)); RF_TC_ATTR((k_tc_conv_staged_i8<128, true>)); RF_TC_ATTR((k_tc_conv_staged_i8<256, true>));
    RF_TC_ATTR((k_tc_dwpw_staged_i8<32, true>)); RF_TC_ATTR((k_tc_dwpw_staged_i8<64, true>)); RF_TC_ATTR((k_tc_dwpw_staged_i8<128, true>)); RF_TC_ATTR((k_tc_dwpw_staged_i8<256, true>));
    RF_TC_ATTR((k_tc_dwpw_staged_i8<32, false>)); RF_TC_ATTR((k_tc_dwpw_staged_i8<64, false>)); RF_TC_ATTR((k_tc_dwpw_staged_i8<128, false>)); RF_TC_ATTR((k_tc_dwpw_staged_i8<256, false>));
    RF_TC_ATTR(k_tc_dwpw_2d_i8<32>); RF_TC_ATTR(k_tc_dwpw_2d_i8<64>); RF_TC_ATTR(k_tc_dwpw_2d_i8<128>); RF_TC_ATTR(k_tc_dwpw_2d_i8<256>);
#undef RF_TC_ATTR
    return cudaSuccess;
}

// ---- INT8 operations: the tensor-core kernels on int8 activations, every tensor's scale looked up by its name -------------------
struct I8Ops : PlanOps {
    using PlanOps::PlanOps;
    static int8_t *q(rf_handle h, const Run &r, int id) { return reinterpret_cast<int8_t *>(r.ctx.arena + h->tensors[id].offset); }
    float scale_of(const std::string &name) const {
        auto it = B.h->int8_scales.find(name);
        if (it == B.h->int8_scales.end()) throw PlanFail{RF_ERR_MODEL, "INT8 calibration table lacks the scale of tensor '" + name + "'"};
        return it->second;
    }
    float tscale(int id) const { return scale_of(B.h->tensors[id].name); }

    // FP32 inside, the output quantised with the scale of relu2
    int stem(const StemNode &n) override { return plan_stem_fused<int8_t>(B, n, "_i8", 1.0f / scale_of(n.pair.out)); }

    int pair(const PairNode &p, int tin) override {
        rf_handle h = B.h;
        auto Wd = [h](size_t off) { return h->d_weights + off; };
        const FoldedConv &dw = *p.dw, &pw = *p.pw;
        const int i = p.i, C = dw.cout, S = dw.stride, N = pw.cout;
        const int ih = p.h, iw = p.w, oh = ih / S, ow_ = iw / S;
        const float s_in = tscale(tin), s_mid = scale_of(p.mid);
        size_t owd = B.add_weights(pack_dw(dw, s_in)), obd = B.add_weights(dw.b);     // float32 products, as the oracle
        const int Kpad = (C + 31) / 32 * 32;
        const DwGeom geo = dw_geometry(C, N, ih, iw, S, [C, Kpad](int rows, int Ns, int R) {
            TcDwArgsI8 a{};
            a.C = C; a.Rmax = R; a.Kpad = Kpad; a.N = Ns; a.rows = rows;
            return R <= TC_MAX_R && tc_dw_i8_smem_bytes(a) <= (size_t)TC_SMEM_LIMIT;
        });
        if (geo.rows == 0) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("INT8 layer %s (%dx%d, %d channels) does not fit shared memory", dw.name.c_str(), iw, ih, C)};
        int tpw = B.tensor(p.out, oh, ow_, N);
        std::vector<float> s_out(N, tscale(tpw));
        QWeights qw = pack_tc_weights_i8({&pw}, s_mid, s_out, Kpad / 16, geo.nsplit);
        size_t oimg = B.add_weights_q(qw.img), omul = B.add_weights(qw.mult), obq = B.add_weights(qw.bq);
        const float inv_mid = 1.0f / s_mid;
        Step s;
        s.name = fmt("i8_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
        s.in = {tin}; s.out = {tpw};
        s.flops_per_img = 2.0 * oh * ow_ * C * 9 + 2.0 * oh * ow_ * C * N;
        s.bytes_per_img = (double)ih * iw * C + (double)oh * ow_ * N;
        const int tw = dw2d_tile_w(h, C, oh, ow_, geo.nsplit);
        if (tw) {
            s.name = fmt("i8_2d_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
            TcDw2dArgsI8 g{};
            g.OH = oh; g.OW = ow_; g.S = S; g.TH = 8; g.TW = tw;
            tc_dw2d_i8_finish(g);
            s.geom = fmt("TH=%d TW=%d OH=%d OW=%d tiles_x=%d tiles_y=%d", g.TH, g.TW, oh, ow_, g.tiles_x, g.tiles_y);
        } else {
            s.geom = fmt("rows=%d nsplit=%d Rmax=%d OH=%d OW=%d", geo.rows, geo.nsplit, geo.Rmax, oh, ow_);
        }
        s.launch = [=](const Run &r) {
            if (tw) {
                TcDw2dArgsI8 a{};
                a.in = q(h, r, tin); a.C = C; a.nimg = r.n; a.IH = ih; a.IW = iw; a.OH = oh; a.OW = ow_; a.S = S; a.N = N; a.Kpad = Kpad;
                a.TH = 8; a.TW = tw;
                tc_dw2d_i8_finish(a);
                a.wimg = h->d_weights_q + oimg; a.mult = Wd(omul); a.bq = Wd(obq); a.dw_w = Wd(owd); a.dw_b = Wd(obd); a.inv_mid = inv_mid;
                a.out = q(h, r, tpw);
                launch_tc_dwpw_2d_i8(a, r.stream);
                return;
            }
            TcDwArgsI8 a{};
            a.in = q(h, r, tin); a.C = C; a.nimg = r.n; a.IH = ih; a.IW = iw; a.OH = oh; a.OW = ow_; a.S = S;
            a.N = N / geo.nsplit; a.Ntotal = N; a.Kpad = Kpad; a.rows = geo.rows; a.Wp = iw + 2; a.Hp = ih + 1; a.Rmax = geo.Rmax;
            a.wimg = h->d_weights_q + oimg; a.mult = Wd(omul); a.bq = Wd(obq); a.dw_w = Wd(owd); a.dw_b = Wd(obd); a.inv_mid = inv_mid;
            a.out = q(h, r, tpw);
            launch_tc_dwpw_i8(a, geo.nsplit, r.stream);
        };
        B.step(std::move(s));
        return tpw;
    }

    void conv(const ConvNode &c) override {
        rf_handle h = B.h;
        auto Wd = [h](size_t off) { return h->d_weights + off; };
        const int cin = c.cs[0]->cin, ks = c.cs[0]->k, tin = c.in, ih = c.h, iw = c.w, tup = c.up;
        const ConvOut o0 = c.out[0], o1 = c.out[1];
        int N = 0;
        for (auto cv : c.cs) N += cv->cout;
        std::vector<float> s_out(N);
        for (int n = 0; n < N; n++) s_out[n] = n < o0.n ? tscale(o0.t) : tscale(o1.t);
        // with the FPN merge fused in, the conv's input tensor is the (never materialised) sum: its scale is the table's
        const float s_in = tup >= 0 ? scale_of(c.sum) : tscale(tin);
        QWeights qw = pack_tc_weights_i8(c.cs, s_in, s_out, tc_i8_gs(cin), 1);
        size_t oimg = B.add_weights_q(qw.img), omul = B.add_weights(qw.mult), obq = B.add_weights(qw.bq);
        size_t oup = 0;
        float lat_mul = 0.f;
        if (tup >= 0) {
            std::vector<float> wq(16 * cin);
            const float s_up = tscale(tup);
            for (int ch = 0; ch < cin; ch++)
                for (int t = 0; t < 16; t++) wq[t * cin + ch] = (float)((double)h->model.up_w[c.up_which][ch * 16 + t] * (double)s_up / (double)s_in);
            oup = B.add_weights(wq);
            lat_mul = (float)((double)tscale(tin) / (double)s_in);
        }
        Step s;
        s.name = "i8_" + c.name;
        s.lane = c.lane;
        s.in = {tin};
        if (tup >= 0) s.in.push_back(tup);
        s.out = {o0.t};
        if (o1.t >= 0) s.out.push_back(o1.t);
        s.flops_per_img = 2.0 * ih * iw * cin * ks * ks * N;
        s.bytes_per_img = (double)ih * iw * cin + (double)ih * iw * N + (tup >= 0 ? (double)(ih / 2) * (iw / 2) * cin : 0.0);
        s.geom = fmt("NT=%d BM=128 H=%d W=%d Hp=%d Wp=%d merge=%s", tc_n_bucket(N), ih, iw, ks == 3 ? ih + 1 : ih, ks == 3 ? iw + 2 : iw,
                     tup >= 0 ? "fused" : "none");
        s.launch = [=](const Run &r) {
            TcConvArgsI8 a{};
            a.in = q(h, r, tin); a.Cin = cin; a.nimg = r.n; a.H = ih; a.W = iw; a.taps = ks * ks; a.N = N;
            a.Wp = ks == 3 ? iw + 2 : iw; a.Hp = ks == 3 ? ih + 1 : ih;
            a.R = (ks == 3 ? 128 + 2 * (iw + 3) : 128) | 1;
            a.wimg = h->d_weights_q + oimg; a.mult = Wd(omul); a.bq = Wd(obq);
            a.out = TcOutI8{q(h, r, o0.t) + o0.off, o0.ld, o0.n, o0.relu, o1.t >= 0 ? q(h, r, o1.t) + o1.off : nullptr, o1.ld, o1.relu};
            if (tup >= 0) { a.up = q(h, r, tup); a.up_wq = Wd(oup); a.lat_mul = lat_mul; a.Cmax = (((a.R / a.Wp + 2) / 2 + 3) * (iw / 2)) | 1; }
            launch_tc_conv_i8(a, r.stream);
        };
        B.step(std::move(s));
    }

    int merge(const MergeNode &m) override {
        rf_handle h = B.h;
        const int tlat = m.lat, tup = m.up, fh = m.h, fw = m.w;
        int plus = B.tensor(m.sum, fh, fw, 64);
        const float s_out = tscale(plus), s_up = tscale(tup), s_lat = tscale(tlat);
        std::vector<float> wq(16 * 64);
        for (int c = 0; c < 64; c++)
            for (int t = 0; t < 16; t++) wq[t * 64 + c] = (float)((double)h->model.up_w[m.level - 1][c * 16 + t] * (double)s_up / (double)s_out);
        size_t owq = B.add_weights(wq);
        const float lat_mul = (float)((double)s_lat / (double)s_out);
        Step s;
        s.name = "i8_fpn_merge_" + m.lv + "_upsample+add";
        s.in = {tlat, tup}; s.out = {plus};
        s.flops_per_img = 2.0 * fh * fw * 64 * 4;
        s.bytes_per_img = (double)fh * fw * 64 * 2 + (double)(fh / 2) * (fw / 2) * 64;
        s.launch = [=](const Run &r) {
            CK(launch_k(k_fpn_merge_i8, dim3((unsigned)((fw * 4 + 127) / 128), (unsigned)fh, (unsigned)r.n), dim3(128), 0, r.stream, (const int8_t *)q(h, r, tlat),
                        (const int8_t *)q(h, r, tup), q(h, r, plus), h->d_weights + owq, lat_mul, r.n, fh, fw, 64));
        };
        B.step(std::move(s));
        return plus;
    }

    // the c2 merge always fused; the c1 merge by the one-wave rule
    bool fuse_merge(const MergeNode &m) override { return m.level == 1 || aggr_fits_one_wave(B.h, m.h, m.w); }

    // FP32 predictors + decode on the dequantised concat tensors, and NMS
    void heads(const HeadsNode &n) override {
        const float s[3] = {tscale(B.h->feat_tensor[0]), tscale(B.h->feat_tensor[1]), tscale(B.h->feat_tensor[2])};
        plan_heads<int8_t>(B, n, s, "i8_");
    }
};

void build_plan_i8(rf_handle h) {
    I8Ops ops(h);
    walk_network(ops);
}

}  // namespace rf_eng

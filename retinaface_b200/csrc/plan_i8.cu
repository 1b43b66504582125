// plan_i8.cu -- the INT8 layer plan of the engine (RF_PREC_INT8).
#include "engine_internal.cuh"
#include "kernels_simt.cuh"
#include "stem_tc.cuh"
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
#define RF_I8C(NT_) if (a.up) launch_k(k_tc_conv_staged_i8<NT_, true>, grid, dim3(TC_THREADS), smem, s, a); else launch_k(k_tc_conv_staged_i8<NT_, false>, grid, dim3(TC_THREADS), smem, s, a)
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
        case 32: launch_k(k_tc_dwpw_2d_i8<32>, grid, dim3(TC_THREADS), smem, s, a); break;
        case 64: launch_k(k_tc_dwpw_2d_i8<64>, grid, dim3(TC_THREADS), smem, s, a); break;
        case 128: launch_k(k_tc_dwpw_2d_i8<128>, grid, dim3(TC_THREADS), smem, s, a); break;
        default: launch_k(k_tc_dwpw_2d_i8<256>, grid, dim3(TC_THREADS), smem, s, a); break;
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
        case 32: if (a.C >= 64) launch_k(k_tc_dwpw_staged_i8<32, true>, grid, dim3(TC_THREADS), smem, s, a); else launch_k(k_tc_dwpw_staged_i8<32, false>, grid, dim3(TC_THREADS), smem, s, a); break;
        case 64: if (a.C >= 64) launch_k(k_tc_dwpw_staged_i8<64, true>, grid, dim3(TC_THREADS), smem, s, a); else launch_k(k_tc_dwpw_staged_i8<64, false>, grid, dim3(TC_THREADS), smem, s, a); break;
        case 128: if (a.C >= 64) launch_k(k_tc_dwpw_staged_i8<128, true>, grid, dim3(TC_THREADS), smem, s, a); else launch_k(k_tc_dwpw_staged_i8<128, false>, grid, dim3(TC_THREADS), smem, s, a); break;
        default: if (a.C >= 64) launch_k(k_tc_dwpw_staged_i8<256, true>, grid, dim3(TC_THREADS), smem, s, a); else launch_k(k_tc_dwpw_staged_i8<256, false>, grid, dim3(TC_THREADS), smem, s, a); break;
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

DwGeom dw_geometry_i8(int C, int N, int IH, int IW, int S) {
    const int OH = IH / S, OW = IW / S, Wp = IW + 2, Hp = IH + 1, Kpad = (C + 31) / 32 * 32;
    auto centre = [&](long m) { long ox = m % OW, oy = (m / OW) % OH, b = m / ((long)OW * OH); return (b * Hp + oy * S) * Wp + ox * S + 1; };
    for (int rows : {128, 64}) {
        if (rows == 128 && OH * OW <= 28 * 28) continue;
        for (int nsplit : {1, 2, 4}) {
            if ((N / nsplit) % 16) continue;
            long g = rows, t = (long)OH * OW;
            while (t) { long u = g % t; g = t; t = u; }
            const long M = ((long)rows / g + 1) * OH * OW;
            int R = 0;
            for (long m0 = 0; m0 < M; m0 += rows) {
                long ml = std::min(m0 + rows, M) - 1;
                R = std::max(R, (int)(centre(ml) - centre(m0) + 2 * (Wp + 1) + 1));
            }
            R |= 1;
            TcDwArgsI8 a{};
            a.C = C; a.Rmax = R; a.Kpad = Kpad; a.N = N / nsplit; a.rows = rows;
            if (R <= TC_MAX_R && tc_dw_i8_smem_bytes(a) <= (size_t)TC_SMEM_LIMIT) return {rows, nsplit, R};
        }
    }
    return {0, 0, 0};
}

void build_plan_i8(rf_handle h) {
    Builder B{h, h->cfg.net_h, h->cfg.net_w};
    const Model &m = h->model;
    const int H = h->cfg.net_h, W = h->cfg.net_w;
    auto Q_ = [h](const Run &r, int id) { return reinterpret_cast<int8_t *>(r.ctx.arena + h->tensors[id].offset); };
    auto Wd = [h](size_t off) { return h->d_weights + off; };
    auto scale_of = [h](const std::string &name) -> float {
        auto it = h->int8_scales.find(name);
        if (it == h->int8_scales.end()) throw PlanFail{RF_ERR_MODEL, "INT8 calibration table lacks the scale of tensor '" + name + "'"};
        return it->second;
    };
    auto tscale = [&](int id) { return scale_of(h->tensors[id].name); };

    // ---- stem: FP32 inside, output quantised with s(relu2) ---------------------------------------------------
    int cur_h = H / 2, cur_w = W / 2;
    int cur = B.tensor("mobilenet0_relu2_fwd", cur_h, cur_w, 16);
    {
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
        const float inv = 1.0f / tscale(cur);
        int out = cur;
        Step s;
        s.name = "stem_conv0+dw1+pw2_u8_to_16ch_i8";
        s.out = {out};
        s.flops_per_img = 2.0 * cur_h * cur_w * (8 * 27 + 8 * 9 + 8 * 16);
        s.bytes_per_img = (double)H * W * 3 + (double)cur_h * cur_w * 16;
        // conv0 on tensor cores, depthwise + pointwise in FP32 on CUDA cores (stem_tc.cuh, OutT = int8_t); RF_FLAG_SIMT_STEM:
        // all three layers on CUDA cores (k_stem)
        const bool simt_stem = (h->cfg.flags & (RF_FLAG_SIMT_STEM | RF_FLAG_NO_TENSORCORE)) != 0;
        size_t oblob = B.add_weights_h(make_stem_blob(w0, c0.b, wd, dw.b, wp, pw.b));
        if (!simt_stem) s.name = "tc_stem_conv0+dw1+pw2_u8_to_16ch_i8";
        const int tiles = ((H / 2 + 15) / 16) * ((W / 2 + 15) / 16);
        const int resident = simt_stem ? 0 : resident_ctas(h, (const void *)k_stem_tc<int8_t>, 256, 0);
        s.launch = [=](const Run &r) {
            if (simt_stem) {
                StemWeights sw{Wd(ow0), Wd(ob0), Wd(owd), Wd(obd), Wd(owp), Wd(obp)};
                launch_k(k_stem<int8_t>, dim3((unsigned)(tiles * r.n)), dim3(256), 0, r.stream, (const PostParams *)r.ctx.d_params, Q_(r, out), sw, r.n, H, W, inv);
            } else {
                StemTcArgs a{reinterpret_cast<const unsigned char *>(h->d_weights_h + oblob)};
                const PersistentGrid pg = persistent_grid(tiles * r.n, resident);
                stem_tc_finish(a, H, W, pg.run);
                launch_k(k_stem_tc<int8_t>, dim3((unsigned)pg.grid), dim3(256), 0, r.stream,
                         (const PostParams *)r.ctx.d_params, Q_(r, out), a, r.n, H, W, inv);
            }
        };
        B.step(std::move(s));
    }
    // ---- 12 x (depthwise + pointwise) --------------------------------------------------------------------------
    int c1 = -1, c2 = -1, c3 = -1;
    for (int i = 3; i <= 26; i += 2) {
        const FoldedConv &dw = m.conv("mobilenet0_conv" + std::to_string(i) + "_fwd");
        const FoldedConv &pw = m.conv("mobilenet0_conv" + std::to_string(i + 1) + "_fwd");
        const int C = dw.cout, S = dw.stride, N = pw.cout;
        const int ih = cur_h, iw = cur_w, oh = cur_h / S, ow_ = cur_w / S;
        const float s_in = tscale(cur), s_mid = scale_of("mobilenet0_relu" + std::to_string(i) + "_fwd");
        std::vector<float> wd(9 * C);
        for (int c = 0; c < C; c++)
            for (int t = 0; t < 9; t++) wd[t * C + c] = dw.w[(size_t)c * 9 + t] * s_in;     // float32 product, as the oracle
        size_t owd = B.add_weights(wd), obd = B.add_weights(dw.b);
        const DwGeom geo = dw_geometry_i8(C, N, ih, iw, S);
        if (geo.rows == 0) throw PlanFail{RF_ERR_UNSUPPORTED, fmt("INT8 layer mobilenet0_conv%d (%dx%d, %d channels) does not fit shared memory", i, iw, ih, C)};
        int tin = cur;
        int tpw = B.tensor("mobilenet0_relu" + std::to_string(i + 1) + "_fwd", oh, ow_, N);
        const int Kpad = (C + 31) / 32 * 32;
        std::vector<float> s_out(N, tscale(tpw));
        QWeights q = pack_tc_weights_i8({&pw}, s_mid, s_out, Kpad / 16, geo.nsplit);
        size_t oimg = B.add_weights_q(q.img), omul = B.add_weights(q.mult), obq = B.add_weights(q.bq);
        const float inv_mid = 1.0f / s_mid;
        Step s;
        s.name = fmt("i8_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
        s.in = {tin}; s.out = {tpw};
        s.flops_per_img = 2.0 * oh * ow_ * C * 9 + 2.0 * oh * ow_ * C * N;
        s.bytes_per_img = (double)ih * iw * C + (double)oh * ow_ * N;
        const bool tiles2d = oh * ow_ > 56 * 56 && C >= 16 && C <= 64 && geo.nsplit == 1 && !(h->cfg.flags & RF_FLAG_DW_1D);   // as the FP16 plan
        if (tiles2d) s.name = fmt("i8_2d_dw%d+pw%d_s%d_%dto%d", i, i + 1, S, C, N);
        s.launch = [=](const Run &r) {
            if (tiles2d) {
                TcDw2dArgsI8 a{};
                a.in = Q_(r, tin); a.C = C; a.nimg = r.n; a.IH = ih; a.IW = iw; a.OH = oh; a.OW = ow_; a.S = S; a.N = N; a.Kpad = Kpad;
                a.TH = 8;
                a.TW = (ow_ + 13) / 14 < (ow_ + 15) / 16 ? 14 : 16;
                tc_dw2d_i8_finish(a);
                a.wimg = h->d_weights_q + oimg; a.mult = Wd(omul); a.bq = Wd(obq); a.dw_w = Wd(owd); a.dw_b = Wd(obd); a.inv_mid = inv_mid;
                a.out = Q_(r, tpw);
                launch_tc_dwpw_2d_i8(a, r.stream);
                return;
            }
            TcDwArgsI8 a{};
            a.in = Q_(r, tin); a.C = C; a.nimg = r.n; a.IH = ih; a.IW = iw; a.OH = oh; a.OW = ow_; a.S = S;
            a.N = N / geo.nsplit; a.Ntotal = N; a.Kpad = Kpad; a.rows = geo.rows; a.Wp = iw + 2; a.Hp = ih + 1; a.Rmax = geo.Rmax;
            a.wimg = h->d_weights_q + oimg; a.mult = Wd(omul); a.bq = Wd(obq); a.dw_w = Wd(owd); a.dw_b = Wd(obd); a.inv_mid = inv_mid;
            a.out = Q_(r, tpw);
            launch_tc_dwpw_i8(a, geo.nsplit, r.stream);
        };
        B.step(std::move(s));
        cur = tpw; cur_h = oh; cur_w = ow_;
        if (i + 1 == 10) c1 = cur;
        if (i + 1 == 22) c2 = cur;
        if (i + 1 == 26) c3 = cur;
    }
    // ---- FPN + SSH ------------------------------------------------------------------------------------------------
    auto conv_step = [&](const std::string &sname, std::vector<const FoldedConv *> cs, int tin, int ih, int iw, int t0, int ld0, int off0,
                         int n0, int relu0, int t1, int ld1, int off1, int relu1, int lane, int tup, int up_which, int tlat_for_up) {
        (void)tlat_for_up;
        const int cin = cs[0]->cin, ks = cs[0]->k;
        int N = 0;
        for (auto c : cs) N += c->cout;
        std::vector<float> s_out(N);
        for (int n = 0; n < N; n++) s_out[n] = n < n0 ? tscale(t0) : tscale(t1);
        // with the FPN merge fused in, the conv's input tensor is the (never materialised) sum: its scale is the table's
        const float s_in = tup >= 0 ? scale_of(up_which == 0 ? "_plus0" : "_plus1") : tscale(tin);
        QWeights q = pack_tc_weights_i8(cs, s_in, s_out, tc_i8_gs(cin), 1);
        size_t oimg = B.add_weights_q(q.img), omul = B.add_weights(q.mult), obq = B.add_weights(q.bq);
        size_t oup = 0;
        float lat_mul = 0.f;
        if (tup >= 0) {
            std::vector<float> wq(16 * cin);
            const float s_up = tscale(tup);
            for (int c = 0; c < cin; c++)
                for (int t = 0; t < 16; t++) wq[t * cin + c] = (float)((double)m.up_w[up_which][c * 16 + t] * (double)s_up / (double)s_in);
            oup = B.add_weights(wq);
            lat_mul = (float)((double)tscale(tin) / (double)s_in);
        }
        Step s;
        s.name = "i8_" + sname;
        s.lane = lane;
        s.in = {tin};
        if (tup >= 0) s.in.push_back(tup);
        s.out = {t0};
        if (t1 >= 0) s.out.push_back(t1);
        s.flops_per_img = 2.0 * ih * iw * cin * ks * ks * N;
        s.bytes_per_img = (double)ih * iw * cin + (double)ih * iw * N + (tup >= 0 ? (double)(ih / 2) * (iw / 2) * cin : 0.0);
        s.launch = [=](const Run &r) {
            TcConvArgsI8 a{};
            a.in = Q_(r, tin); a.Cin = cin; a.nimg = r.n; a.H = ih; a.W = iw; a.taps = ks * ks; a.N = N;
            a.Wp = ks == 3 ? iw + 2 : iw; a.Hp = ks == 3 ? ih + 1 : ih;
            a.R = (ks == 3 ? 128 + 2 * (iw + 3) : 128) | 1;
            a.wimg = h->d_weights_q + oimg; a.mult = Wd(omul); a.bq = Wd(obq);
            a.out = TcOutI8{Q_(r, t0) + off0, ld0, n0, relu0, t1 >= 0 ? Q_(r, t1) + off1 : nullptr, ld1, relu1};
            if (tup >= 0) { a.up = Q_(r, tup); a.up_wq = Wd(oup); a.lat_mul = lat_mul; a.Cmax = (((a.R / a.Wp + 2) / 2 + 3) * (iw / 2)) | 1; }
            launch_tc_conv_i8(a, r.stream);
        };
        B.step(std::move(s));
    };
    auto move_last_step_after_producer = [&](int tensor_id) {
        int pos = 0;
        for (int i = (int)h->steps.size() - 2; i >= 0 && !pos; i--)
            for (int t : h->steps[i].out) if (t == tensor_id) { pos = i + 1; break; }
        Step st = std::move(h->steps.back());
        h->steps.pop_back();
        h->steps.insert(h->steps.begin() + pos, std::move(st));
    };
    auto ssh = [&](const std::string &lvname, int tin, int fh, int fw, int level, int lane) {
        const std::string p = "rf_" + lvname + "_det";
        int cat = B.tensor(p + "_concat_relu", fh, fw, 64);
        int ctx1 = B.tensor(p + "_context_conv1_relu", fh, fw, 16);
        int ctx31 = B.tensor(p + "_context_conv3_1_relu", fh, fw, 16);
        conv_step("ssh_" + lvname + "_conv1+ctx1_3x3_64to48", {&m.conv(p + "_conv1"), &m.conv(p + "_context_conv1")}, tin, fh, fw, cat, 64, 0, 32, 1,
                  ctx1, 16, 0, 1, lane, -1, 0, -1);
        conv_step("ssh_" + lvname + "_ctx2+ctx3_1_3x3_16to32", {&m.conv(p + "_context_conv2"), &m.conv(p + "_context_conv3_1")}, ctx1, fh, fw, cat,
                  64, 32, 16, 1, ctx31, 16, 0, 1, lane, -1, 0, -1);
        conv_step("ssh_" + lvname + "_ctx3_2_3x3_16to16", {&m.conv(p + "_context_conv3_2")}, ctx31, fh, fw, cat, 64, 48, 16, 1, -1, 0, 0, 0, lane, -1,
                  0, -1);
        h->feat_tensor[level] = cat;
    };
    const int h32 = H / 32, w32 = W / 32, h16 = H / 16, w16 = W / 16, h8 = H / 8, w8 = W / 8;
    int lat3 = B.tensor("rf_c3_lateral_relu", h32, w32, 64);
    int lat2 = B.tensor("rf_c2_lateral_relu", h16, w16, 64);
    int lat1 = B.tensor("rf_c1_red_conv_relu", h8, w8, 64);
    conv_step("c1_red_1x1_64to64", {&m.conv("rf_c1_red_conv")}, c1, h8, w8, lat1, 64, 0, 64, 1, -1, 0, 0, 0, 1, -1, 0, -1);
    move_last_step_after_producer(c1);
    conv_step("c2_lateral_1x1_128to64", {&m.conv("rf_c2_lateral")}, c2, h16, w16, lat2, 64, 0, 64, 1, -1, 0, 0, 0, 2, -1, 0, -1);
    move_last_step_after_producer(c2);
    conv_step("c3_lateral_1x1_256to64", {&m.conv("rf_c3_lateral")}, c3, h32, w32, lat3, 64, 0, 64, 1, -1, 0, 0, 0, 0, -1, 0, -1);
    ssh("c3", lat3, h32, w32, 0, 1);
    int aggr2 = B.tensor("rf_c2_aggr_relu", h16, w16, 64);
    conv_step("c2_upsample+add+aggr_3x3_64to64", {&m.conv("rf_c2_aggr")}, lat2, h16, w16, aggr2, 64, 0, 64, 1, -1, 0, 0, 0, 0, lat3, 0, lat2);
    ssh("c2", aggr2, h16, w16, 1, 2);
    int aggr1 = B.tensor("rf_c1_aggr_relu", h8, w8, 64);
    const long c1_tiles = ((long)h->cfg.max_batch * (h8 + 1) * (w8 + 2) + 127) / 128;
    if (c1_tiles <= h->num_sms) {
        conv_step("c1_upsample+add+aggr_3x3_64to64", {&m.conv("rf_c1_aggr")}, lat1, h8, w8, aggr1, 64, 0, 64, 1, -1, 0, 0, 0, 0, aggr2, 1, lat1);
    } else {
        int plus1 = B.tensor("_plus1", h8, w8, 64);
        const float s_out = tscale(plus1), s_up = tscale(aggr2), s_lat = tscale(lat1);
        std::vector<float> wq(16 * 64);
        for (int c = 0; c < 64; c++)
            for (int t = 0; t < 16; t++) wq[t * 64 + c] = (float)((double)m.up_w[1][c * 16 + t] * (double)s_up / (double)s_out);
        size_t owq = B.add_weights(wq);
        const float lat_mul = (float)((double)s_lat / (double)s_out);
        Step s;
        s.name = "i8_fpn_merge_c1_upsample+add";
        s.in = {lat1, aggr2}; s.out = {plus1};
        s.flops_per_img = 2.0 * h8 * w8 * 64 * 4;
        s.bytes_per_img = (double)h8 * w8 * 64 * 2 + (double)(h8 / 2) * (w8 / 2) * 64;
        s.launch = [=](const Run &r) {
            launch_k(k_fpn_merge_i8, dim3((unsigned)((w8 * 4 + 127) / 128), (unsigned)h8, (unsigned)r.n), dim3(128), 0, r.stream, (const int8_t *)Q_(r, lat1), (const int8_t *)Q_(r, aggr2), Q_(r, plus1),
                     Wd(owq), lat_mul, r.n, h8, w8, 64);
        };
        B.step(std::move(s));
        conv_step("c1_aggr_3x3_64to64", {&m.conv("rf_c1_aggr")}, plus1, h8, w8, aggr1, 64, 0, 64, 1, -1, 0, 0, 0, 0, -1, 0, -1);
    }
    ssh("c1", aggr1, h8, w8, 2, 0);
    // ---- predictors + decode (FP32 on the dequantised concat tensors) and NMS -------------------------------------
    size_t hw_off[3], hb_off[3];
    float hs[3];
    const int strides[3] = {32, 16, 8};
    for (int l = 0; l < 3; l++) {
        std::string st = "_stride" + std::to_string(strides[l]);
        const FoldedConv *cs[3] = {&m.conv("face_rpn_cls_score" + st), &m.conv("face_rpn_bbox_pred" + st), &m.conv("face_rpn_landmark_pred" + st)};
        std::vector<float> w(32 * 64), b(32);
        int r = 0;
        for (auto c : cs)
            for (int o = 0; o < c->cout; o++, r++) {
                b[r] = c->b[o];
                for (int ci = 0; ci < 64; ci++) w[r * 64 + ci] = c->w[(size_t)o * 64 + ci];
            }
        hw_off[l] = B.add_weights(w);
        hb_off[l] = B.add_weights(b);
        hs[l] = tscale(h->feat_tensor[l]);
    }
    {
        Step s;
        s.name = "i8_heads_1x1+softmax+decode_all_levels";
        s.in = {h->feat_tensor[0], h->feat_tensor[1], h->feat_tensor[2]};
        double px = (double)h32 * w32 + (double)h16 * w16 + (double)h8 * w8;
        s.flops_per_img = 2.0 * px * 64 * 4;
        s.bytes_per_img = px * 64;
        int f0 = h->feat_tensor[0], f1 = h->feat_tensor[1], f2 = h->feat_tensor[2];
        size_t w0 = hw_off[0], w1 = hw_off[1], w2 = hw_off[2], b0 = hb_off[0], b1 = hb_off[1], b2 = hb_off[2];
        float s0 = hs[0], s1 = hs[1], s2 = hs[2];
        s.launch = [=](const Run &r) {
            const int8_t *feat[3] = {Q_(r, f0), Q_(r, f1), Q_(r, f2)};
            HeadWeights hws[3] = {{Wd(w0), Wd(b0), s0}, {Wd(w1), Wd(b1), s1}, {Wd(w2), Wd(b2), s2}};
            launch_head_decode<int8_t>(feat, hws, h->lv, r.n, W, H, r.ctx.d_params, r.ctx.pb, r.blobs, r.stream, true);
        };
        s.name = "i8_heads_1x1+softmax+decode+nms_all_levels";      // decode -> NMS in one launch (last block per image)
        h->head_step = (int)h->steps.size();
        B.step(std::move(s));
    }
}

// Cross-lane dependencies: a step waits (event) for the producers of its inputs that live in another lane.
}  // namespace rf_eng

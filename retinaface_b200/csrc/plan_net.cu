// plan_net.cu -- the network every layer plan is built from: one walk of the reference's graph (model/mnet-deconv-0517.prototxt)
// in step order, calling the operations of one plan (PlanOps: SIMT in plan_fp.cu, FP16 tensor cores in plan_tile.cu, INT8 in
// plan_i8.cu).  The walk knows the layer and tensor names, the shapes, the lanes and the order; the operations know the kernels.
#include "engine_internal.cuh"

namespace rf_eng {

// ---- the walk ---------------------------------------------------------------------------------------------------------------
// Lanes: the forward graph is not a chain.  rf_c1_red_conv only needs C1 and rf_c2_lateral only C2, so they run on side lanes
// while the backbone continues, and each is emitted right after the step that produces its input: the step list, which the
// arena's liveness analysis walks in order, must show a side-lane step where it may start.  Each level's SSH runs on a side lane
// while the main lane walks the top-down path lat3 -> aggr2 -> aggr1 -> ssh_c1 (the critical path).
void walk_network(PlanOps &ops) {
    Builder &B = ops.B;
    rf_handle h = B.h;
    const Model &m = h->model;
    auto conv = [&](const std::string &name) { return &m.conv(name); };
    auto pair_node = [&](int i, int ih, int iw) {
        return PairNode{i, conv(fmt("mobilenet0_conv%d_fwd", i)), conv(fmt("mobilenet0_conv%d_fwd", i + 1)), fmt("mobilenet0_relu%d_fwd", i),
                        fmt("mobilenet0_relu%d_fwd", i + 1), ih, iw};
    };
    int fh = h->cfg.net_h / 2, fw = h->cfg.net_w / 2;
    int cur = ops.stem(StemNode{conv("mobilenet0_conv0_fwd"), "mobilenet0_relu0_fwd", pair_node(1, fh, fw)});

    // ---- 12 x (depthwise 3x3, pointwise 1x1) in six segments, C1 / C2 / C3 and their lateral convs (prototxt:55-1192) --------
    struct Seg { std::vector<int> pairs; const char *lat, *step; int lane; };
    const Seg segs[6] = {{{3, 5}, nullptr, nullptr, 0},
                         {{7, 9}, "rf_c1_red_conv", "c1_red_1x1_64to64", 1},
                         {{11, 13, 15}, nullptr, nullptr, 0},
                         {{17, 19, 21}, "rf_c2_lateral", "c2_lateral_1x1_128to64", 2},
                         {{23}, nullptr, nullptr, 0},
                         {{25}, "rf_c3_lateral", "c3_lateral_1x1_256to64", 0}};
    int lat[3] = {-1, -1, -1}, lh[3] = {0, 0, 0}, lw[3] = {0, 0, 0};     // per FPN level, 0 = stride 32
    for (int k = 0; k < 6; k++) {
        SegNode s;
        for (int i : segs[k].pairs) {
            s.pairs.push_back(pair_node(i, fh, fw));
            fh /= s.pairs.back().dw->stride; fw /= s.pairs.back().dw->stride;
        }
        if (segs[k].lat) {
            s.lat.name = segs[k].step; s.lat.cs = {conv(segs[k].lat)}; s.lat.h = fh; s.lat.w = fw; s.lat.lane = segs[k].lane;
            s.lat.out[0] = ConvOut{-1, 64, 0, 64, 1};
            s.lat_out = std::string(segs[k].lat) + "_relu";
        }
        const SegOut o = ops.segment(s, cur);
        cur = o.out;
        if (segs[k].lat) { const int l = 2 - k / 2; lat[l] = o.lat; lh[l] = fh; lw[l] = fw; }
    }

    // ---- FPN top-down + SSH (prototxt:1199-2302) ------------------------------------------------------------------------------
    const char *lvn[3] = {"c3", "c2", "c1"};
    HeadsNode heads{};
    auto ssh = [&](int l, int in, int lane) {
        const std::string p = std::string("rf_") + lvn[l] + "_det", st = fmt("_stride%d", 32 >> l);
        for (int q = 0; q < 3; q++)
            heads.pred[l][q] = conv((q == 0 ? "face_rpn_cls_score" : q == 1 ? "face_rpn_bbox_pred" : "face_rpn_landmark_pred") + st);
        const int cat = B.tensor(p + "_concat_relu", lh[l], lw[l], 64);
        h->feat_tensor[l] = cat;
        ops.ssh(SshNode{lvn[l], p + "_context_conv1_relu", p + "_context_conv3_1_relu", l, lane, in, lh[l], lw[l], cat, conv(p + "_conv1"),
                        conv(p + "_context_conv1"), conv(p + "_context_conv2"), conv(p + "_context_conv3_1"), conv(p + "_context_conv3_2"),
                        {heads.pred[l][0], heads.pred[l][1], heads.pred[l][2]}});
    };
    auto merge_aggr = [&](int l, int up) {
        const std::string lv = lvn[l];
        const int aggr = B.tensor("rf_" + lv + "_aggr_relu", lh[l], lw[l], 64);
        MergeNode mn{lv, fmt("_plus%d", l - 1), l, lat[l], up, lh[l], lw[l], {}, {}};
        mn.aggr.name = lv + "_aggr_3x3_64to64"; mn.aggr.cs = {conv("rf_" + lv + "_aggr")}; mn.aggr.h = lh[l]; mn.aggr.w = lw[l];
        mn.aggr.out[0] = ConvOut{aggr, 64, 0, 64, 1};
        mn.fused = mn.aggr;
        mn.fused.name = lv + "_upsample+add+aggr_3x3_64to64"; mn.fused.in = lat[l];
        mn.fused.up = up; mn.fused.up_which = l - 1; mn.fused.sum = mn.sum;
        ops.merge_aggr(mn);
        return aggr;
    };
    ssh(0, lat[0], 1);
    const int aggr2 = merge_aggr(1, lat[0]);
    ssh(1, aggr2, 2);
    const int aggr1 = merge_aggr(2, aggr2);
    ssh(2, aggr1, 0);
    ops.heads(heads);
}

// ---- default graph-level operations from the leaves -------------------------------------------------------------------------
SegOut PlanOps::segment(const SegNode &s, int in) {
    for (const PairNode &p : s.pairs) in = pair(p, in);
    if (s.lat.cs.empty()) return {in, -1};
    ConvNode c = s.lat;
    c.in = in;
    c.out[0].t = B.tensor(s.lat_out, c.h, c.w, 64);
    conv(c);
    return {in, c.out[0].t};
}

void PlanOps::merge_aggr(const MergeNode &m) {
    if (fuse_merge(m)) return conv(m.fused);
    ConvNode c = m.aggr;
    c.in = merge(m);
    conv(c);
}

void PlanOps::ssh(const SshNode &n) {
    const int ctx1 = B.tensor(n.ctx1, n.h, n.w, 16), ctx31 = B.tensor(n.ctx31, n.h, n.w, 16);
    auto node = [&](const char *name, std::vector<const FoldedConv *> cs, int in, int off, int n0, int t1) {
        ConvNode c;
        c.name = "ssh_" + n.lv + name; c.cs = std::move(cs); c.in = in; c.h = n.h; c.w = n.w; c.lane = n.lane;
        c.out[0] = ConvOut{n.cat, 64, off, n0, 1};
        if (t1 >= 0) c.out[1] = ConvOut{t1, 16, 0, 16, 1};
        return c;
    };
    // det_conv1 (64->32, ReLU after the concat) + context_conv1 (64->16): one launch
    conv(node("_conv1+ctx1_3x3_64to48", {n.conv1, n.ctx_conv1}, n.in, 0, 32, ctx1));
    // context_conv2 (16->16 -> concat[32:48]) + context_conv3_1 (16->16): one launch
    conv(node("_ctx2+ctx3_1_3x3_16to32", {n.ctx_conv2, n.ctx_conv3_1}, ctx1, 32, 16, ctx31));
    // context_conv3_2 (16->16 -> concat[48:64])
    conv(node("_ctx3_2_3x3_16to16", {n.ctx_conv3_2}, ctx31, 48, 16, -1));
}

// ---- leaf helpers the plans share ---------------------------------------------------------------------------------------------
StemPack pack_stem(const StemNode &n) {
    const FoldedConv &c0 = *n.conv0, &dw = *n.pair.dw, &pw = *n.pair.pw;
    StemPack p{std::vector<float>(27 * 8), std::vector<float>(72), std::vector<float>(128)};
    for (int o = 0; o < 8; o++)
        for (int cb = 0; cb < 3; cb++)       // cb: BGR channel of the u8 image; network channel = 2 - cb (RGB)
            for (int t = 0; t < 9; t++) p.w0[(t * 3 + cb) * 8 + o] = c0.w[((size_t)o * 3 + (2 - cb)) * 9 + t];
    for (int c = 0; c < 8; c++)
        for (int t = 0; t < 9; t++) p.wd[t * 8 + c] = dw.w[(size_t)c * 9 + t];
    for (int o = 0; o < 16; o++)
        for (int c = 0; c < 8; c++) p.wp[c * 16 + o] = pw.w[(size_t)o * 8 + c];
    return p;
}

std::vector<float> pack_dw(const FoldedConv &dw, float scale) {
    const int C = dw.cout;
    std::vector<float> wd(9 * C);
    for (int c = 0; c < C; c++)
        for (int t = 0; t < 9; t++) wd[t * C + c] = dw.w[(size_t)c * 9 + t] * scale;
    return wd;
}

// Tile geometry of one fused depthwise+pointwise layer: rows per CTA, N slices and the exact upper bound of the staged range,
// so that everything fits in shared memory.  fits(rows, N / nsplit, R): the kernel takes that geometry.
DwGeom dw_geometry(int C, int N, int IH, int IW, int S, const std::function<bool(int rows, int N, int R)> &fits) {
    const int OH = IH / S, OW = IW / S, Wp = IW + 2, Hp = IH + 1;
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
            if (fits(rows, N / nsplit, R)) return {rows, nsplit, R};
        }
    }
    return {0, 0, 0};
}

// Large maps (> 56x56 outputs; measured: no gain below): 2-D tiles (tc_dwpw2d.cuh, tc_dwpw2d_i8.cuh) -- half the staged halo,
// no position table, vertical reuse.  8 rows by the width of 14 or 16 that needs fewer tiles per row.
int dw2d_tile_w(rf_handle h, int C, int oh, int ow, int nsplit) {
    if (oh * ow <= 56 * 56 || C < 16 || C > 64 || nsplit != 1 || (h->cfg.flags & RF_FLAG_DW_1D)) return 0;
    return (ow + 13) / 14 < (ow + 15) / 16 ? 14 : 16;
}

// Fusing the merge into the aggr conv costs ~50 KB of shared memory: fine while the conv's tiles fit one wave (c2 level), a loss
// once it forces a second wave (c1 level at batch 8: 207 tiles, 1 CTA/SM).
bool aggr_fits_one_wave(rf_handle h, int fh, int fw) {
    return ((long)h->cfg.max_batch * (fh + 1) * (fw + 2) + 127) / 128 <= h->num_sms;
}

}  // namespace rf_eng

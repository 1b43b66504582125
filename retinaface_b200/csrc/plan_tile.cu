// plan_tile.cu -- the FP16 tensor-core layer plan: which parts of the network walk (plan_net.cu) run as stages of which
// persistent tile-chain kernel (tile_chain.cuh), the shared-memory budget of every chain, the packed weights, the TMA tensor
// maps.  Chains run only on a handle with one execution context (TileOps); everything else, and every chain that does not
// fit (wide maps), runs on the per-layer tensor-core kernels of plan_fp.cu, layer by layer.
//
//   stem, backbone, laterals        per-layer kernels (k_stem_tc, k_tc_dwpw_staged / k_tc_dwpw_2d, k_tc_conv_staged)
//   tile_<lv>_merge+aggr            FPN merge (lateral + upsampled coarser level) + aggr 3x3          (c2, c1; max_batch <= 2)
//   tile_ssh_<lv>[+heads+decode]    SSH det/context convs [+ predictors + decode + last-block NMS]     (c3, c2, c1)
#include "engine_internal.cuh"
#include "tile_chain.cuh"

namespace rf_eng {

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

constexpr int TCH_SMEM_LIMIT = 226 * 1024;    // dynamic shared memory a chain may use (227 KB per CTA minus the static part)

// NHWC FP16 tensor [n][H][W][C] as a 4-D map {C, W, H, n}; box {bc, bw, bh, 1}; element strides {1, es, es, 1};
// swizzle mode by the bytes of one box row (bc * 2: 32 / 64 / 128)
CUtensorMap make_map(const void *base, int C, int W, int H, int n, int bc, int bw, int bh, int es) {
    CUtensorMap m;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {(cuuint32_t)bc, (cuuint32_t)bw, (cuuint32_t)bh, 1};
    cuuint32_t est[4] = {1, (cuuint32_t)es, (cuuint32_t)es, 1};
    const CUtensorMapSwizzle sw = bc * 2 == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (bc * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(base), dims, strides, box, est, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw PlanFail{RF_ERR_CUDA, fmt("cuTensorMapEncodeTiled failed (%d) for a %dx%dx%d tensor, box %dx%dx%d", (int)r, C, W, H, bc, bw, bh)};
    return m;
}

int round_up(int v, int a) { return (v + a - 1) / a * a; }

}  // namespace

// Host description of one chain: logical buffers + stages (ChainSpec), then the finalised kernel arguments.
struct TileChain {
    struct LBuf {
        int C = 0;
        int halo = 0;                 // rows beyond the tile the consumers need, each side
        bool stored = false;          // the owned rows are TMA-stored into an arena tensor ...
        int store_tensor = -1;        // ... this one (assigned once the chain is known to fit)
        int first = 1 << 30, last = -1;   // stage indices (input: first = -1)
        bool is_merge = false;
    };
    struct LStage {
        int type = TCH_CONV, Cin = 0, N = 0, taps = 1, in_buf = 0;
        std::vector<int> ob_buf, ob_c16, ob_relu;
        std::vector<__half> wp_img;
        std::vector<float> bp;
        int hs = 0;
        int store_buf = -1;
        double flops = 0;             // per output position
    };
    std::string name;
    std::vector<LBuf> bufs;
    std::vector<LStage> stages;
    int in_tensor = -1, in_C = 0, in_W = 0, in_H = 0;   // chain input (arena tensor) and its map size
    int W = 0, H = 0;                 // resolution the chain works at
    int merge_tensor = -1;            // FPN merge: coarser level (64 channels, W/2 x H/2)
    std::vector<__half> merge_w;      // [16 taps][64]
    int level = -1;                   // TCH_HEAD (predictors + decode + last-block NMS): FPN level (0: stride 32)
    // finalised
    TchArgs args{};
    size_t bias_off = 0;              // float offset into d_weights
    int store_buf_of[3] = {-1, -1, -1}, store_C[3] = {0, 0, 0};     // store map i <- logical buffer
    int nstores = 0;
    int TH = 0, mtiles = 0;           // rows per tile, MMA tiles per CTA tile (cost proxy)
};

namespace {

// ---- chain construction helpers ----------------------------------------------------------------------------------------
int add_buf(TileChain &c, int C, bool stored = false, int store_tensor = -1) {
    TileChain::LBuf b;
    b.C = C;
    b.stored = stored;
    b.store_tensor = store_tensor;
    c.bufs.push_back(b);
    return (int)c.bufs.size() - 1;
}

// convolution (all `cs` share the input and are concatenated along N); per conv: destination buffer, channel offset, ReLU
struct ConvDst { int buf, coff, relu; };
int add_conv(TileChain &c, int in_buf, const std::vector<const FoldedConv *> &cs, const std::vector<ConvDst> &dst) {
    TileChain::LStage s;
    s.type = TCH_CONV; s.Cin = cs[0]->cin; s.taps = cs[0]->k * cs[0]->k; s.in_buf = in_buf;
    int Kpad = 0;
    s.wp_img = pack_tc_weights(cs, s.bp, Kpad);
    s.N = (int)s.bp.size();
    for (size_t i = 0; i < cs.size(); i++)
        for (int j = 0; j < cs[i]->cout / 16; j++) { s.ob_buf.push_back(dst[i].buf); s.ob_c16.push_back(dst[i].coff / 16 + j); s.ob_relu.push_back(dst[i].relu); }
    s.flops = 2.0 * s.Cin * s.taps * s.N;
    c.stages.push_back(std::move(s));
    return (int)c.stages.size() - 1;
}

// the three predictor convs of one level as one N = 32 GEMM with hi + lo FP16 weight pieces (FP32-grade products)
int add_head(TileChain &c, int in_buf, const FoldedConv *const cs[3]) {
    TileChain::LStage s;
    s.type = TCH_HEAD; s.Cin = 64; s.N = 32; s.taps = 1; s.in_buf = in_buf;
    std::vector<__half> hi((size_t)64 * 32), lo((size_t)64 * 32);
    int r = 0;
    for (int q = 0; q < 3; q++)
        for (int o = 0; o < cs[q]->cout; o++, r++) {
            s.bp.push_back(cs[q]->b[o]);
            for (int ci = 0; ci < 64; ci++) {
                const float w = cs[q]->w[(size_t)o * 64 + ci];
                const __half wh = __float2half(w);
                hi[((size_t)(ci / 8) * 32 + r) * 8 + ci % 8] = wh;
                lo[((size_t)(ci / 8) * 32 + r) * 8 + ci % 8] = __float2half(w - __half2float(wh));
            }
        }
    s.wp_img = hi;
    s.wp_img.insert(s.wp_img.end(), lo.begin(), lo.end());
    s.flops = 2.0 * 64 * 32 * 2;
    c.stages.push_back(std::move(s));
    return (int)c.stages.size() - 1;
}

// ---- finalisation: halos, rows, shared-memory placement, kernel arguments --------------------------------------------------
// returns false when the chain does not fit with TH rows per tile
bool finalize_chain(rf_handle h, TileChain &c, int TH, int max_faces, bool resident) {
    const int ns = (int)c.stages.size(), nb = (int)c.bufs.size();
    if (ns > TCH_MAX_STAGES || nb > TCH_MAX_BUFS) return false;
    const int Wl = c.W + 2;
    if (Wl > 256) return false;
    // halos (reverse stage order: all consumers of a buffer come after its producers)
    for (auto &b : c.bufs) { b.halo = 0; b.first = 1 << 30; b.last = -1; }
    for (int s = ns - 1; s >= 0; s--) {
        auto &st = c.stages[s];
        int hs = 0;
        for (int b : st.ob_buf) hs = std::max(hs, c.bufs[b].halo);
        st.hs = hs;
        c.bufs[st.in_buf].halo = std::max(c.bufs[st.in_buf].halo, hs + (st.taps == 9 ? 1 : 0));
    }
    const int HT = c.bufs[0].halo;       // buffer 0 is the chain input
    // lifetimes
    c.bufs[0].first = -1;
    for (int b = 0; b < nb; b++) if (c.bufs[b].is_merge) { c.bufs[b].first = -1; c.bufs[b].last = -1; }
    for (int s = 0; s < ns; s++) {
        auto &st = c.stages[s];
        c.bufs[st.in_buf].last = std::max(c.bufs[st.in_buf].last, s);
        for (int b : st.ob_buf) { c.bufs[b].first = std::min(c.bufs[b].first, s); c.bufs[b].last = std::max(c.bufs[b].last, s); }
    }
    for (auto &b : c.bufs) if (b.stored) b.last = ns;     // TMA stores read the buffer until the next tile starts
    if (c.merge_tensor >= 0) c.bufs[0].last = std::max(c.bufs[0].last, 0);

    TchArgs &a = c.args;
    a = TchArgs{};
    a.nstages = ns; a.nbufs = nb;
    a.Wl = Wl; a.HT = HT; a.TH = TH;
    a.W = c.W; a.H = c.H;
    a.tiles_per_img = (c.H + TH - 1) / TH;
    a.in_C = c.in_C;
    // buffers
    std::vector<int> bytes(nb);
    for (int b = 0; b < nb; b++) {
        auto &lb = c.bufs[b];
        TchBuf &tb = a.buf[b];
        tb.row = lb.C >= 64 ? 128 : lb.C * 2;
        tb.slabs = std::max(1, lb.C / 64);
        tb.rows_lo = HT - lb.halo;
        tb.nrows = TH + 2 * lb.halo;
        // positions in front of the first row: the (-1, -1) tap of the first computed position reads one back; TMA-loaded
        // buffers need their row 0 128-byte aligned (8), TMA-stored ones their position (row, lx = 1) (7 for rows < 128 bytes)
        tb.slack = (lb.stored && tb.row < 128) ? 7 : 8;
        if (lb.is_merge) {
            a.merge_rows = (TH + 2 * HT) / 2 + 3;
            tb.rows_lo = 0; tb.nrows = a.merge_rows;
            tb.slab_stride = round_up(a.merge_rows * (c.W / 2 + 2) * 128, 1024);
            bytes[b] = tb.slab_stride;
            continue;
        }
        tb.slab_stride = round_up((tb.slack + tb.nrows * Wl + 8) * tb.row, 1024);
        bytes[b] = tb.slabs * tb.slab_stride;
        if (b == 0) a.in_bytes = (unsigned)tb.slabs * (unsigned)(std::min(lb.C, 64) * 2 * Wl * tb.nrows);
    }
    if (c.merge_tensor >= 0) a.merge_bytes = (unsigned)(64 * 2 * (c.W / 2 + 2) * a.merge_rows);
    // first-fit placement by first use
    std::vector<int> order(nb);
    for (int i = 0; i < nb; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return c.bufs[x].first < c.bufs[y].first; });
    std::vector<int> placed;
    int top = 0;
    for (int id : order) {
        int off = 0;
        bool moved = true;
        while (moved) {
            moved = false;
            for (int p : placed) {
                const bool live = !(c.bufs[p].last < c.bufs[id].first || c.bufs[id].last < c.bufs[p].first);
                const bool mem = off < a.buf[p].off + bytes[p] && a.buf[p].off < off + bytes[id];
                if (live && mem) { off = a.buf[p].off + bytes[p]; moved = true; }
            }
        }
        a.buf[id].off = off;
        top = std::max(top, off + bytes[id]);
        placed.push_back(id);
    }
    // stages
    int wp_max = 0, read_end = 0, mt = 0;
    std::vector<float> bias;
    for (int s = 0; s < ns; s++) {
        auto &ls = c.stages[s];
        TchStage &st = a.st[s];
        st.type = ls.type; st.Cin = ls.Cin; st.N = ls.N; st.taps = ls.taps; st.in_buf = ls.in_buf;
        st.rows_lo = HT - ls.hs; st.nrows = TH + 2 * ls.hs;
        if ((int)ls.ob_buf.size() > 16 || ls.N % 16 || ls.Cin % 16 || ls.N > 256) return false;
        for (size_t j = 0; j < ls.ob_buf.size(); j++) { st.ob_buf[j] = (unsigned char)ls.ob_buf[j]; st.ob_c16[j] = (unsigned char)ls.ob_c16[j]; st.ob_relu[j] = (unsigned char)ls.ob_relu[j]; }
        st.wp_bytes = (int)ls.wp_img.size() * 2;
        wp_max = std::max(wp_max, st.wp_bytes);
        st.bias_pw = (int)bias.size(); bias.insert(bias.end(), ls.bp.begin(), ls.bp.end());
        while (bias.size() % 4) bias.push_back(0.f);
        st.store_buf = -1; st.store_map = -1;
        // furthest byte a (partial) MMA tile of this stage may read: rows past the range + one tap
        const TchBuf &bi = a.buf[ls.in_buf];
        const int ntile = (st.nrows * Wl + 127) / 128;
        mt += ntile;
        const int pos0 = bi.slack + (st.rows_lo - bi.rows_lo) * Wl;
        read_end = std::max(read_end, bi.off + (bi.slabs - 1) * bi.slab_stride + (pos0 + ntile * 128 + Wl + 2) * bi.row);
    }
    c.mtiles = mt;
    // a stage's outputs are stored once the LAST stage writing the buffer is complete
    c.nstores = 0;
    for (int b = 0; b < nb; b++) {
        if (!c.bufs[b].stored) continue;
        if (c.nstores == 3) return false;
        int last_writer = -1;
        for (int s = 0; s < ns; s++) for (int ob : c.stages[s].ob_buf) if (ob == b) last_writer = s;
        if (last_writer < 0 || a.st[last_writer].store_buf >= 0) return false;
        a.st[last_writer].store_buf = b; a.st[last_writer].store_map = c.nstores;
        c.store_buf_of[c.nstores] = b; c.store_C[c.nstores] = c.bufs[b].C;
        // TMA store sources (position (row, lx = 1) of every owned row) must be 128-byte aligned
        if (((a.buf[b].slack + 1) * a.buf[b].row) % 128 || (Wl * a.buf[b].row) % 128) return false;
        c.nstores++;
    }
    if (c.merge_tensor >= 0) {
        a.merge_C = 64;
        for (int b = 0; b < nb; b++) if (c.bufs[b].is_merge) a.merge_buf = b;
        a.merge_w_bias = (int)bias.size();
        const float *mw = reinterpret_cast<const float *>(c.merge_w.data());
        bias.insert(bias.end(), mw, mw + c.merge_w.size() / 2);
    }
    // weights, bias arena, NMS scratch behind the buffers
    const int nms_need = c.level >= 0 ? (int)((sizeof(NmsSmem) + 15) / 16 * 16 + sizeof(int) * (size_t)max_faces) : 0;
    a.resident = resident ? 1 : 0;
    int cursor = round_up(top, 1024);
    if (resident) {
        // every stage keeps its own weight region for the CTA's lifetime
        for (int s = 0; s < ns; s++) { a.st[s].wp_smem = cursor; cursor += round_up(a.st[s].wp_bytes, 128); }
        a.wp_smem = cursor;
        // NMS scratch: the input tile's region (dead by then, never TMA-stored) when large enough
        if (nms_need && bytes[0] >= nms_need) a.head.nms_smem = a.buf[0].off;
        else { a.head.nms_smem = cursor; cursor += round_up(nms_need, 128); }
    } else {
        a.wp_smem = cursor; cursor += std::max(round_up(wp_max, 128), round_up(nms_need, 128));
        a.head.nms_smem = a.wp_smem;
    }
    a.bias_smem = cursor;
    a.bias_floats = (int)bias.size();
    a.smem_bytes = std::max(a.bias_smem + a.bias_floats * 4, read_end) + 1024;      // + alignment slack of the dynamic base
    if (a.smem_bytes > TCH_SMEM_LIMIT) return false;
    c.TH = TH;
    c.bias_off = (size_t)-1;
    // (weights go to the handle's arenas once the geometry is final: commit_chain)
    c.args.bias_floats = (int)bias.size();
    // stash the bias vector in the chain until commit
    h->tile_bias_tmp = bias;
    return true;
}

// copies the packed weights + bias arena of a finalised chain into the handle's upload staging
void commit_chain(Builder &B, TileChain &c) {
    rf_handle h = B.h;
    for (size_t s = 0; s < c.stages.size(); s++) c.args.st[s].wp_off = (int)(B.add_weights_h(c.stages[s].wp_img) * 2);
    c.bias_off = B.add_weights(h->tile_bias_tmp);
}

// picks the tile height: among the heights that fit, the one with the least (waves x MMA tiles per CTA), ties to the taller
bool choose_tile(rf_handle h, TileChain &c, int max_batch, int max_faces) {
    double best = 1e30;
    int best_th = 0;
    bool best_res = false;
    for (int th = 1; th <= std::min(c.H, 32); th++) {
        for (int res = 1; res >= 0; res--) {
            if (!finalize_chain(h, c, th, max_faces, res != 0)) continue;
            const long tiles = (long)max_batch * c.args.tiles_per_img;
            // k_tile_chain's register budget allows one CTA per SM, and its grid is one CTA per SM
            const double waves = std::ceil((double)tiles / h->num_sms);
            // MMA tiles + per-stage hand-offs (streamed weights: one exposed load per stage) + per-tile set-up
            const double cost = waves * (c.mtiles + (res ? 1.0 : 4.0) * c.stages.size() + 4.0);
            if (cost < best || (cost == best && th > best_th)) { best = cost; best_th = th; best_res = res != 0; }
            break;      // resident fits: no need to look at streaming for this height
        }
    }
    if (!best_th) return false;
    return finalize_chain(h, c, best_th, max_faces, best_res);
}

void launch_chain(rf_handle h, const std::shared_ptr<TileChain> &cp, const Run &r) {
    const int n = r.n;
    cudaStream_t st = r.stream;
    TileChain &c = *cp;
    TchArgs a = c.args;
    a.nimg = n;
    a.ntiles = n * a.tiles_per_img;
    a.dbg = h->tile_dbg_dev;
    a.trace = nullptr;
#ifdef RF_TCH_TRACE
    {   // one trace buffer per chain (host-mapped), reset at every launch: holds the LAST launch's timeline of CTA 0
        static std::map<const TileChain *, unsigned long long *> bufs;
        auto it = bufs.find(&c);
        if (it == bufs.end()) {
            unsigned long long *p = nullptr;
            CK(cudaHostAlloc(&p, 8 * 1024, cudaHostAllocMapped));
            it = bufs.emplace(&c, p).first;
        }
        CK(cudaStreamSynchronize(st));
        if (it->second[0]) {
            const unsigned n = (unsigned)std::min<unsigned long long>(it->second[0], 500);
            fprintf(stderr, "TRACE %s:", c.name.c_str());
            for (unsigned i = 0; i < n; i++) fprintf(stderr, " %llu@%llu", it->second[1 + 2 * i], it->second[2 + 2 * i] - it->second[2]);
            fprintf(stderr, "\n");
        }
        memset(it->second, 0, 8 * 1024);
        a.trace = it->second;
    }
#endif
    a.warena = reinterpret_cast<const unsigned char *>(h->d_weights_h);
    a.bias = h->d_weights + c.bias_off;
    TchMaps maps;
    memset(&maps, 0, sizeof maps);
    const TchBuf &b0 = a.buf[0];
    const int bc = std::min(c.in_C, 64);
    auto T_ = [&](int id) { return r.ctx.arena + h->tensors[id].offset; };
    maps.in = make_map(T_(c.in_tensor), c.in_C, c.in_W, c.in_H, n, bc, a.Wl, b0.nrows, 1);
    if (c.merge_tensor >= 0) maps.aux = make_map(T_(c.merge_tensor), 64, c.W / 2, c.H / 2, n, 64, c.W / 2 + 2, a.merge_rows, 1);
    for (int i = 0; i < c.nstores; i++) maps.st[i] = make_map(T_(c.bufs[c.store_buf_of[i]].store_tensor), c.store_C[i], c.W, c.H, n, std::min(c.store_C[i], 64), c.W, 1, 1);
    if (c.level >= 0) {
        a.head.lv = h->lv[c.level];
        a.head.pb = r.ctx.pb;
        a.head.params = r.ctx.d_params;
        a.head.net_w = h->cfg.net_w; a.head.net_h = h->cfg.net_h;
        a.head.done = r.ctx.pb.tile_done;
        a.head.expected = r.single ? 0 : h->tile_expected;    // a step launched on its own: no last-block NMS
        for (int k = 0; k < 3; k++) a.head.blobs[k] = r.blobs ? r.blobs[3 * c.level + k] : nullptr;
    }
    const int grid = std::min(a.ntiles, h->num_sms);
    CK(launch_k(k_tile_chain<0>, dim3((unsigned)grid), dim3(TCH_THREADS), (size_t)a.smem_bytes, st, maps, a));
}

// adds the step of a finalised chain
void add_chain_step(Builder &B, std::shared_ptr<TileChain> c, int lane, double bytes_per_img) {
    rf_handle h = B.h;
    commit_chain(B, *c);
    h->chains.push_back(c);
    Step s;
    s.name = c->name;
    s.lane = lane;
    s.in = {c->in_tensor};
    if (c->merge_tensor >= 0) s.in.push_back(c->merge_tensor);
    for (int i = 0; i < c->nstores; i++) s.out.push_back(c->bufs[c->store_buf_of[i]].store_tensor);
    double fl = 0;
    for (auto &ls : c->stages) fl += ls.flops * c->W * c->H;
    s.flops_per_img = fl;
    s.bytes_per_img = bytes_per_img;
    s.geom = fmt("TH=%d H=%d W=%d tiles_per_img=%d weights=%s", c->TH, c->H, c->W, c->args.tiles_per_img, c->args.resident ? "resident" : "streamed");
    s.launch = [h, c](const Run &r) { launch_chain(h, c, r); };
    B.step(std::move(s));
}

}  // namespace

// one line per chain: geometry, budgets (for rf_plan_describe and the CPU-side planner tests)
std::string describe_chains(rf_handle h) {
    std::string out;
    for (auto &cp : h->chains) {
        const TileChain &c = *cp;
        const TchArgs &a = c.args;
        out += fmt("%s: %dx%d map, TH=%d HT=%d Wl=%d, %d tiles/image, %d stages, %d MMA tiles/tile, smem %d B (%s weights), stores %d\n",
                   c.name.c_str(), c.W, c.H, a.TH, a.HT, a.Wl, a.tiles_per_img, a.nstages, c.mtiles, a.smem_bytes, a.resident ? "resident" : "streamed",
                   c.nstores);
    }
    return out;
}

cudaError_t tile_init() {
    if (!g_encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
        if (e != cudaSuccess) return e;
        if (!fn) return cudaErrorNotSupported;
        g_encode = (EncodeTiledFn)fn;
    }
    return cudaFuncSetAttribute(k_tile_chain<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCH_SMEM_LIMIT);
}

// The FP16 tensor-core plan.  With ONE execution context (a single forward at a time: the blocking / latency mode) the SSH
// chains with the predictors, decode and last-block NMS fused in (and, at batch 1-2, the merge + aggr chains) save launches
// and round trips through memory (tools/plan_sweep.py measures them against the per-layer kernels); with several contexts
// overlapping batches (throughput mode) what counts is SM time per step, where the per-layer kernels win -- there only the
// fused decode + NMS tail is taken over.  Every part without a chain, or whose chain does not fit, runs per layer.
struct TileOps : PlanOps {
    const bool ssh_chains, chain_heads, aggr_chains;
    std::shared_ptr<TileChain> ssh_chain[3];                  // the SSH chains: the last-block NMS needs all three
    bool split_heads = false;                                 // some level's predictors are fused, others not: no plan
    TileOps(rf_handle h, bool chains, bool with_heads)
        : PlanOps(h), ssh_chains(chains), chain_heads(chains && with_heads), aggr_chains(chains && h->cfg.max_batch <= 2) {}
    int stem(const StemNode &n) override { return plan_stem_fused<__half>(B, n, "", 1.0f); }
    int pair(const PairNode &p, int in) override { return plan_pair_tc(B, p, in); }
    void conv(const ConvNode &c) override { plan_conv_tc(B, c); }
    int merge(const MergeNode &m) override { return plan_fpn_merge_h2(B, m); }
    bool fuse_merge(const MergeNode &m) override { return aggr_fits_one_wave(B.h, m.h, m.w); }

    // merged = lat + upsample(up); aggr 3x3 64->64
    void merge_aggr(const MergeNode &m) override {
        rf_handle h = B.h;
        if (!aggr_chains) return PlanOps::merge_aggr(m);
        auto c = std::make_shared<TileChain>();
        c->name = "tile_" + m.lv + "_merge+aggr";
        c->in_tensor = m.lat; c->in_C = 64; c->in_W = m.w; c->in_H = m.h;
        c->W = m.w; c->H = m.h;
        c->merge_tensor = m.up;
        c->merge_w.resize(16 * 64);
        for (int ch = 0; ch < 64; ch++)
            for (int t = 0; t < 16; t++) c->merge_w[t * 64 + ch] = __float2half(h->model.up_w[m.level - 1][ch * 16 + t]);
        int bi = add_buf(*c, 64);
        int bm = add_buf(*c, 64);
        c->bufs[bm].is_merge = true;
        int bo = add_buf(*c, 64, true, m.aggr.out[0].t);
        add_conv(*c, bi, m.aggr.cs, {{bo, 0, 1}});
        if (!choose_tile(h, *c, h->cfg.max_batch, h->cfg.max_faces)) return PlanOps::merge_aggr(m);
        add_chain_step(B, c, 0, ((double)m.h * m.w * 64 * 2 + (double)(m.h / 2) * (m.w / 2) * 64) * 2);
    }

    void ssh(const SshNode &n) override {
        rf_handle h = B.h;
        if (!ssh_chains) return PlanOps::ssh(n);
        auto c = std::make_shared<TileChain>();
        c->name = "tile_ssh_" + n.lv + (chain_heads ? "+heads+decode" : "");
        c->in_tensor = n.in; c->in_C = 64; c->in_W = n.w; c->in_H = n.h;
        c->W = n.w; c->H = n.h;
        int bi = add_buf(*c, 64);
        int bcat = add_buf(*c, 64, true, n.cat);
        int bctx1 = add_buf(*c, 16);
        int bctx31 = add_buf(*c, 16);
        // branches that share an input run as ONE stage over the rows the neediest branch wants: an MMA's time is its A-operand
        // read from shared memory (128 rows x 32 bytes whatever N), so the other branch's output columns ride along for free
        add_conv(*c, bi, {n.conv1, n.ctx_conv1}, {{bcat, 0, 1}, {bctx1, 0, 1}});
        add_conv(*c, bctx1, {n.ctx_conv2, n.ctx_conv3_1}, {{bcat, 32, 1}, {bctx31, 0, 1}});
        add_conv(*c, bctx31, {n.ctx_conv3_2}, {{bcat, 48, 1}});
        if (chain_heads) {
            add_head(*c, bcat, n.pred);
            c->level = n.level;
        }
        if (!choose_tile(h, *c, h->cfg.max_batch, h->cfg.max_faces)) return PlanOps::ssh(n);
        add_chain_step(B, c, n.lane, ((double)n.h * n.w * 64 * 2) * 2);
        ssh_chain[n.level] = c;
    }

    void heads(const HeadsNode &n) override {
        rf_handle h = B.h;
        const float one[3] = {1.f, 1.f, 1.f};
        if (!(ssh_chain[0] && ssh_chain[1] && ssh_chain[2] && chain_heads)) {
            // some level's predictors are not fused: none may be (one decode kernel covers all levels)
            for (auto &c : ssh_chain)
                if (c && c->level >= 0) split_heads = true;
            if (!split_heads) plan_heads<__half>(B, n, one, "");
            return;
        }
        h->tile_expected = ssh_chain[0]->args.tiles_per_img + ssh_chain[1]->args.tiles_per_img + ssh_chain[2]->args.tiles_per_img;
    }
};

void build_plan_tiles(rf_handle h) {
    // the chains are meant for one forward at a time AND small batches; at large batches every per-layer kernel fills the GPU.
    // RF_FLAG_LEGACY_TC: no chains.
    const bool chains = h->cfg.streams == 1 && h->cfg.max_batch <= 16 && !(h->cfg.flags & RF_FLAG_LEGACY_TC);
    for (bool with_heads : {true, false}) {        // predictors fused into some SSH chains but not all: again without
        // a failed attempt leaves no trace
        h->steps.clear(); h->tensors.clear(); h->tensor_by_name.clear(); h->chains.clear();
        h->wstage.clear(); h->wstage_h.clear(); h->wstage_q.clear();
        h->tile_expected = 0;
        for (int &f : h->feat_tensor) f = -1;
        TileOps ops(h, chains, with_heads);
        walk_network(ops);
        if (!ops.split_heads) return;
    }
    throw PlanFail{RF_ERR_UNSUPPORTED, "no tile-chain plan fits this network size; create the handle with RF_FLAG_LEGACY_TC"};
}

}  // namespace rf_eng

// engine.cu -- the handle behind include/rf_b200.h: model upload, activation arena, CUDA-graph executor and the detect C-ABI
// entry points.  The layer plans live in plan_fp.cu (FP32 / FP16) and plan_i8.cu (INT8), the video tracker in tracker.cu; shared
// types in engine_internal.cuh.
//
// Replaces the reference's engine slot: TrtNetBase / TrtRetinaFaceNet
// (retinaface/tensorrt/trtnetbase.cpp:199-330, trtretinafacenet.cpp:48-210) and the detect
// orchestration of RetinaFace::detect / detectBatchImages (retinaface/RetinaFace.cpp:576-940).
#include <array>
#include <cmath>

#include "engine_internal.cuh"
#include "calibrate.cuh"
#include "preprocess.cuh"

namespace rf_eng {

std::string &create_error() {
    thread_local std::string text;
    return text;
}

// Cross-lane dependencies: a step waits (event) for the producers of its inputs that live in another lane.
void link_steps(rf_handle h) {
    auto &st = h->steps;
    for (int i = 0; i < (int)st.size(); i++) {
        st[i].deps.clear();
        for (int t : st[i].in) {
            for (int j = i - 1; j >= 0; j--) {
                bool writes = false;
                for (int o : st[j].out) writes |= (o == t);
                if (!writes) continue;
                if (st[j].lane != st[i].lane) {
                    if (std::find(st[i].deps.begin(), st[i].deps.end(), j) == st[i].deps.end()) st[i].deps.push_back(j);
                    st[j].signals = true;
                }
                break;   // the last writer before i (its lane orders earlier writers of the same tensor)
            }
        }
    }
    // the forward ends on the main lane: side lanes whose last step nobody waits for (SSH chains with fused predictors)
    // are joined explicitly at the end of run_steps
    for (int l = 1; l < 3; l++) {
        h->lane_last[l] = -1;
        for (int i = 0; i < (int)st.size(); i++) if (st[i].lane == l) h->lane_last[l] = i;
        if (h->lane_last[l] >= 0) st[h->lane_last[l]].signals = true;
    }
}

// Liveness-based first-fit placement of activation tensors in one arena.  Steps on side lanes run
// concurrently with later main-lane steps: every tensor such a step touches stays live until the
// first step of another lane that waits for its lane (the join), so no concurrent writer can land on it.
void place_tensors(rf_handle h, bool keep_all) {
    auto &ts = h->tensors;
    auto &st = h->steps;
    for (int si = 0; si < (int)st.size(); si++) {
        for (int t : st[si].out) { if (ts[t].first < 0) ts[t].first = si; ts[t].last = std::max(ts[t].last, si); }
        for (int t : st[si].in) ts[t].last = std::max(ts[t].last, si);
    }
    for (int k = 0; k < (int)st.size(); k++) {
        if (st[k].lane == 0) continue;
        int join = (int)st.size() - 1;
        for (int j = k + 1; j < (int)st.size() && join == (int)st.size() - 1; j++)
            for (int d : st[j].deps)
                if (st[j].lane != st[k].lane && st[d].lane == st[k].lane && d >= k) { join = j; break; }
        for (int t : st[k].in) ts[t].last = std::max(ts[t].last, join);
        for (int t : st[k].out) ts[t].last = std::max(ts[t].last, join);
    }
    // a main-lane step that runs while a side lane is still reading must not overwrite those inputs either:
    // covered above because the side step's inputs stay live until the join.
    const size_t B = (size_t)h->cfg.max_batch;
    size_t top = 0;
    std::vector<int> order(ts.size());
    for (size_t i = 0; i < ts.size(); i++) order[i] = (int)i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ts[a].first < ts[b].first; });
    std::vector<int> placed;
    for (int id : order) {
        size_t sz = (ts[id].bytes_per_img * B + 255) / 256 * 256;
        size_t off = 0;
        if (keep_all) {
            off = top;
        } else {
            bool moved = true;
            while (moved) {
                moved = false;
                for (int p : placed) {
                    bool live_overlap = !(ts[p].last < ts[id].first || ts[id].last < ts[p].first);
                    size_t psz = (ts[p].bytes_per_img * B + 255) / 256 * 256;
                    bool mem_overlap = off < ts[p].offset + psz && ts[p].offset < off + sz;
                    if (live_overlap && mem_overlap) { off = ts[p].offset + psz; moved = true; }
                }
            }
        }
        ts[id].offset = off;
        top = std::max(top, off + sz);
        placed.push_back(id);
    }
    h->arena_bytes = top;
}

// The layer plan of h->cfg (INT8, FP32, FP16 tile chains or FP16 per-layer kernels), linked across lanes and placed in the
// arena.  `init`: also set the kernels' launch attributes up on the current device (rf_plan_describe needs no GPU).
void make_plan(rf_handle h, bool init) {
    const rf_config &cfg = h->cfg;
    const bool simt = cfg.precision == RF_PREC_FP32 || (cfg.precision == RF_PREC_FP16 && (cfg.flags & RF_FLAG_NO_TENSORCORE));
    h->on_device = init;
    if (init && !simt) CK(tc_init());
    if (cfg.precision == RF_PREC_INT8) { if (init) CK(tc_init_i8()); build_plan_i8(h); }
    else if (cfg.precision == RF_PREC_FP32) build_plan<float>(h);
    else if (simt) build_plan<__half>(h);
    else { if (init) CK(tile_init()); build_plan_tiles(h); }
    link_steps(h);
    place_tensors(h, false);
}

// Candidate and output buffers of the NMS for `batch` images of up to `anchors` candidates each.
void alloc_post_buffers(PostBuffers &pb, int anchors, int batch, int max_faces) {
    int ap2 = 1;
    while (ap2 < anchors) ap2 <<= 1;
    pb.anchors_per_image = anchors; pb.anchors_pow2 = ap2; pb.max_faces = max_faces; pb.max_batch = batch;
    const size_t B = batch;
    CK(cudaMalloc(&pb.cand_keys, sizeof(unsigned long long) * B * anchors));
    CK(cudaMalloc(&pb.cand_recs, sizeof(rf_det) * B * anchors));
    CK(cudaMalloc(&pb.cand_count, sizeof(int) * B));
    CK(cudaMemset(pb.cand_count, 0, sizeof(int) * B));
    CK(cudaMalloc(&pb.sort_scratch, sizeof(unsigned long long) * B * ap2));
    CK(cudaMalloc(&pb.flag_scratch, B * ap2));
    CK(cudaMalloc(&pb.out_dets, sizeof(rf_det) * B * max_faces));
    CK(cudaMalloc(&pb.out_counts, sizeof(int) * B));
    CK(cudaMalloc(&pb.out_total_kept, sizeof(int) * B));
    CK(cudaMemset(pb.out_counts, 0, sizeof(int) * B));
    CK(cudaMalloc(&pb.tile_done, sizeof(int) * B));
    CK(cudaMemset(pb.tile_done, 0, sizeof(int) * B));
}
void free_post_buffers(PostBuffers &pb) {
    cudaFree(pb.cand_keys); cudaFree(pb.cand_recs); cudaFree(pb.cand_count); cudaFree(pb.sort_scratch); cudaFree(pb.flag_scratch);
    cudaFree(pb.out_dets); cudaFree(pb.out_counts); cudaFree(pb.out_total_kept); cudaFree(pb.tile_done);
    pb = PostBuffers{};
}

// Allocates context c's arena (h->arena_bytes); with `all`, everything else the context owns too.
void create_ctx(rf_handle h, Ctx &c, bool all) {
    if (all) {
        CK(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
        for (int l = 1; l < 3; l++) CK(cudaStreamCreateWithFlags(&c.lane_stream[l], cudaStreamNonBlocking));
        c.step_event.assign(h->steps.size(), nullptr);
        for (size_t i = 0; i < h->steps.size(); i++)
            if (h->steps[i].signals) CK(cudaEventCreateWithFlags(&c.step_event[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c.fence, cudaEventDisableTiming));
    }
    CK(cudaMalloc(&c.arena, h->arena_bytes));
    if (!all) return;
    CK(cudaMalloc(&c.d_params, sizeof(PostParams)));
    CK(cudaHostAlloc(&c.h_params, sizeof(PostParams) * Ctx::kParamSlots, cudaHostAllocDefault));
    int anchors = 0;
    for (const LevelDesc &lv : h->lv) anchors += 2 * lv.h * lv.w;
    alloc_post_buffers(c.pb, anchors, h->cfg.max_batch, h->cfg.max_faces);
}

// Waits for context c, drops its captured graphs (they hold arena addresses) and frees its arena; with `all`, everything else
// the context owns too.
void release_ctx(Ctx &c, bool all) {
    if (c.stream) cudaStreamSynchronize(c.stream);
    for (auto &g : c.graphs) cudaGraphExecDestroy(g.second);
    c.graphs.clear();
    cudaFree(c.arena);
    c.arena = nullptr;
    if (!all) return;
    cudaFree(c.d_params); cudaFreeHost(c.h_params); cudaFree(c.d_frames_in); cudaFree(c.d_redact);
    free_post_buffers(c.pb);
    for (auto e : c.step_event) if (e) cudaEventDestroy(e);
    for (int l = 1; l < 3; l++) if (c.lane_stream[l]) cudaStreamDestroy(c.lane_stream[l]);
    if (c.fence) cudaEventDestroy(c.fence);
    if (c.stream) cudaStreamDestroy(c.stream);
    c = Ctx{};
}

// Issue the forward pass into r.ctx: lane 0 on r.stream, side lanes on the context's lane streams, joined by events.  Works
// both under stream capture (the side streams fork from / join into the capturing stream) and eagerly.
void run_steps(rf_handle h, const Run &r, bool use_lanes = true) {
    static const bool one_lane = [] { const char *e = getenv("RF_ONE_LANE"); return e && e[0] == '1'; }();   // A/B measurements
    if (one_lane) use_lanes = false;
    const Ctx &c = r.ctx;
    for (size_t i = 0; i < h->steps.size(); i++) {
        Step &st = h->steps[i];
        cudaStream_t cs = (use_lanes && st.lane) ? c.lane_stream[st.lane] : r.stream;
        if (use_lanes)
            for (int d : st.deps) CK(cudaStreamWaitEvent(cs, c.step_event[d], 0));
        st.launch(Run{c, r.n, cs, r.blobs});
        if (use_lanes && st.signals) CK(cudaEventRecord(c.step_event[i], cs));
    }
    if (use_lanes)
        for (int l = 1; l < 3; l++)
            if (h->lane_last[l] >= 0) CK(cudaStreamWaitEvent(r.stream, c.step_event[h->lane_last[l]], 0));
    // multi-GPU handles: the wait for every rank's records of this step is the forward's last node (a no-op kernel for runs
    // without an exchange), not a separate launch behind the graph
    if (h->comm.ready) comm_wait_in_graph(h, c, r.n, r.stream);
}

void forward_graph(rf_handle h, Ctx &c, int n) {
    if (h->cfg.flags & RF_FLAG_NO_GRAPH) {
        run_steps(h, Run{c, n, c.stream});
        CK(cudaGetLastError());
        return;
    }
    auto it = c.graphs.find(n);
    if (it == c.graphs.end()) {
        cudaGraph_t g = nullptr;
        CK(cudaStreamBeginCapture(c.stream, cudaStreamCaptureModeThreadLocal));
        run_steps(h, Run{c, n, c.stream});
        cudaError_t e = cudaStreamEndCapture(c.stream, &g);
        if (e != cudaSuccess) throw CudaFail{e, "cudaStreamEndCapture", __FILE__, __LINE__};
        cudaGraphExec_t ge = nullptr;
        e = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) throw CudaFail{e, "cudaGraphInstantiate", __FILE__, __LINE__};
        it = c.graphs.emplace(n, ge).first;
    }
    CK(cudaGraphLaunch(it->second, c.stream));
}

// Run parameters travel through a small ring of pinned slots so that an asynchronous caller
// (rf_detect_batch_device) can queue several runs without overwriting a copy still in flight.
void set_params(rf_handle h, Ctx &c, float thr, float nms, const uint8_t *input = nullptr, unsigned comm_seq = 0) {
    PostParams *slot = c.h_params + (c.param_seq++ % Ctx::kParamSlots);
    slot->score_thr = thr;
    slot->nms_thr = nms;
    slot->input = input ? input : h->d_input;
    slot->comm_seq = comm_seq;
    slot->comm_slot = comm_seq ? comm_seq % (unsigned)h->comm.ring : 0u;
    c.cur_thr = thr;
    c.cur_nms = nms;
    CK(cudaMemcpyAsync(c.d_params, slot, sizeof(PostParams), cudaMemcpyHostToDevice, c.stream));
}

void destroy(rf_handle h) {
    if (!h) return;
    cudaSetDevice(h->device);
    for (Ctx &c : h->ctx) if (c.stream) cudaStreamSynchronize(c.stream);
    comm_release(h);
    jpeg_release(h);
    for (Ctx &c : h->ctx) release_ctx(c, true);
    free_post_buffers(h->pb_merge);
    free_post_buffers(h->pb_tiles);
    for (auto *ring : {&h->tiled_slots, &h->rotated_slots})
        for (auto &s : *ring) {
            free_post_buffers(s.pb);
            if (s.free) cudaEventDestroy(s.free);
            if (s.start) cudaEventDestroy(s.start);
        }
    cudaFree(h->d_weights); cudaFree(h->d_weights_h); cudaFree(h->d_weights_q); cudaFree(h->d_input); cudaFree(h->d_raw);
    for (auto p : h->d_blobs) cudaFree(p);
    h->copy_pool.reset();
    for (auto e : h->raw_ev) if (e) cudaEventDestroy(e);
    cudaFree(h->d_align_crops); cudaFree(h->d_align_mats);
    cudaFreeHost(h->h_input); cudaFreeHost(h->h_raw); cudaFreeHost(h->h_dets); cudaFreeHost(h->h_counts); cudaFreeHost(h->tile_dbg);
    for (auto &sl : h->slots) {
        cudaFree(sl.d_in); cudaFreeHost(sl.h_in); cudaFreeHost(sl.h_dets); cudaFreeHost(sl.h_counts);
        if (sl.ev_h2d) cudaEventDestroy(sl.ev_h2d);
        if (sl.ev_done) cudaEventDestroy(sl.ev_done);
    }
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    delete h;
}

int check_n(rf_handle h, int n) {
    if (!h) return RF_ERR_INVALID_ARG;
    if (n < 0) return fail(h, RF_ERR_INVALID_ARG, "negative batch size");
    if (n > h->cfg.max_batch) return fail(h, RF_ERR_CAPACITY, fmt("batch %d exceeds max_batch %d", n, h->cfg.max_batch));
    return RF_OK;
}

}  // namespace rf_eng

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

int rf_abi_version(void) { return RF_B200_ABI_VERSION; }

const char *rf_build_info(void) {
    return "librf_b200 (RetinaFace mnet25 detect path) built for sm_90a, CUDA " RF_STR(CUDART_VERSION);
}

const char *rf_status_string(int s) {
    switch (s) {
        case RF_OK: return "ok";
        case RF_ERR_INVALID_ARG: return "invalid argument";
        case RF_ERR_IO: return "i/o error";
        case RF_ERR_MODEL: return "model error";
        case RF_ERR_CUDA: return "CUDA error";
        case RF_ERR_NO_DEVICE: return "no usable CUDA device (the library has no CPU path)";
        case RF_ERR_CAPACITY: return "capacity exceeded";
        case RF_ERR_UNSUPPORTED: return "unsupported";
    }
    return "unknown status";
}

const char *rf_last_error(rf_handle h) { return h ? h->err.c_str() : create_error().c_str(); }

int rf_create(const rf_config *cfg, rf_handle *out) {
    if (out) *out = nullptr;
    if (!cfg || !out) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_create: cfg and out must be non-NULL");
    if (!cfg->caffemodel_path) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_create: caffemodel_path is NULL");
    rf_config cfg_local = *cfg;
    NetGraph graph;
    Model model;
    int cache_status = CACHE_NONE;
    {
        // model front end first: the prototxt may supply the network size (trtnetbase.cpp:163-187 reads it from there too)
        std::string err;
        int st = RF_OK;
        if (cfg->network) {
            NetworkConfig nc;
            if (!network_config(cfg->network, nc, err)) return fail(nullptr, RF_ERR_UNSUPPORTED, "rf_create: " + err);
            if (nc.ratios.size() != 1) return fail(nullptr, RF_ERR_UNSUPPORTED, fmt("rf_create: network '%s' uses %zu anchor ratios per scale; the shipped models (and this engine) have 2 anchors per position", cfg->network, nc.ratios.size()));
        }
        if (!load_model(cfg->caffemodel_path, cfg->prototxt_path ? cfg->prototxt_path : "", cfg->cache_path ? cfg->cache_path : "", model, &graph, &cache_status, err, st))
            return fail(nullptr, st, err);
        if (cfg->prototxt_path && cfg_local.net_w == 0 && cfg_local.net_h == 0) { cfg_local.net_h = graph.input_dims[2]; cfg_local.net_w = graph.input_dims[3]; }
    }
    cfg = &cfg_local;
    if (cfg->net_w <= 0 || cfg->net_h <= 0 || cfg->net_w % 32 || cfg->net_h % 32)
        return fail(nullptr, RF_ERR_INVALID_ARG, fmt("rf_create: net size %dx%d must be positive multiples of 32", cfg->net_w, cfg->net_h));
    if (cfg->max_batch <= 0 || cfg->max_batch > 4096) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_create: max_batch must be in [1, 4096]");
    {
        // The kernels index activations with 32-bit element offsets (and pack (image row) << 12 | column in the FPN merge):
        // the largest tensor of a batch -- the stem output, (H/2) x (W/2) x 16 -- must stay below 2^31 elements.
        const long long stem_elems = (long long)cfg->max_batch * (cfg->net_h / 2) * (cfg->net_w / 2) * 16;
        const long long merge_rows = (long long)cfg->max_batch * (cfg->net_h / 8);
        if (stem_elems > 0x7fffffffLL || merge_rows >= (1LL << 19) || cfg->net_w / 8 >= (1 << 12))
            return fail(nullptr, RF_ERR_CAPACITY, fmt("rf_create: max_batch %d at %dx%d exceeds the 32-bit activation index range (largest tensor: %lld elements); "
                                                      "use a smaller max_batch", cfg->max_batch, cfg->net_w, cfg->net_h, stem_elems));
    }
    if (cfg->precision != RF_PREC_FP32 && cfg->precision != RF_PREC_FP16 && cfg->precision != RF_PREC_INT8)
        return fail(nullptr, RF_ERR_INVALID_ARG, "rf_create: unknown precision");
    if (cfg->precision == RF_PREC_INT8 && !cfg->int8_table_path)
        return fail(nullptr, RF_ERR_INVALID_ARG, "rf_create: RF_PREC_INT8 needs int8_table_path (the TensorRT calibration cache of this caffemodel)");

    std::unique_ptr<rf_handle_s, void (*)(rf_handle)> H(new rf_handle_s, destroy);
    rf_handle h = H.get();
    h->cfg = *cfg;
    h->caffemodel = cfg->caffemodel_path;
    h->cfg.caffemodel_path = h->caffemodel.c_str();
    if (cfg->int8_table_path) { h->table = cfg->int8_table_path; h->cfg.int8_table_path = h->table.c_str(); }
    if (h->cfg.max_faces <= 0) h->cfg.max_faces = 256;
    if (h->cfg.max_faces > 8192) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_create: max_faces must be <= 8192");
    if (h->cfg.max_image_w <= 0) h->cfg.max_image_w = h->cfg.net_w;
    if (h->cfg.max_image_h <= 0) h->cfg.max_image_h = h->cfg.net_h;
    h->cfg.max_image_w = std::max(h->cfg.max_image_w, h->cfg.net_w);
    h->cfg.max_image_h = std::max(h->cfg.max_image_h, h->cfg.net_h);
    h->device = cfg->device;
    h->elem = cfg->precision == RF_PREC_FP32 ? 4 : (cfg->precision == RF_PREC_FP16 ? 2 : 1);

    // ---- model (host) --------------------------------------------------------------------
    {
        std::string err;
        h->model = std::move(model);
        h->cache_status = cache_status;
        h->cfg.prototxt_path = h->cfg.cache_path = h->cfg.network = nullptr;     // (the caller's strings are not kept)
        if (!h->table.empty() && !read_int8_table(h->table, h->int8_scales, err)) return fail(nullptr, RF_ERR_IO, err);
    }
    // ---- device ----------------------------------------------------------------------------
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, RF_ERR_NO_DEVICE, fmt("no CUDA device (%s); librf_b200 has no CPU path", e == cudaSuccess ? "count 0" : cudaGetErrorString(e)));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, RF_ERR_INVALID_ARG, fmt("device %d out of range (%d devices)", cfg->device, ndev));
    try {
        CK(cudaSetDevice(h->device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, h->device));
        if (prop.major != 9 || prop.minor != 0)
            return fail(nullptr, RF_ERR_NO_DEVICE, fmt("device %d is sm_%d%d; librf_b200 is built for sm_90a only", h->device, prop.major, prop.minor));
        h->num_sms = prop.multiProcessorCount;
        CK(cudaEventCreate(&h->ev0));
        CK(cudaEventCreate(&h->ev1));
        CK(postproc_init());

        const int Hn = h->cfg.net_h, Wn = h->cfg.net_w, Bm = h->cfg.max_batch;
        // levels / anchors
        const int strides[3] = {32, 16, 8};
        int abase = 0, pbase = 0;
        for (int l = 0; l < 3; l++) {
            LevelDesc &lv = h->lv[l];
            lv.stride = strides[l]; lv.h = Hn / strides[l]; lv.w = Wn / strides[l];
            lv.anchor_base = abase; lv.pix_base = pbase;
            base_anchors_net3(strides[l], lv.base);
            abase += 2 * lv.h * lv.w; pbase += lv.h * lv.w;
        }
        make_plan(h, true);
        CK(cudaMalloc(&h->d_weights, h->wstage.size() * sizeof(float)));
        CK(cudaMemcpy(h->d_weights, h->wstage.data(), h->wstage.size() * sizeof(float), cudaMemcpyHostToDevice));
        if (!h->wstage_h.empty()) {
            CK(cudaMalloc(&h->d_weights_h, h->wstage_h.size() * sizeof(__half)));
            CK(cudaMemcpy(h->d_weights_h, h->wstage_h.data(), h->wstage_h.size() * sizeof(__half), cudaMemcpyHostToDevice));
        }
        if (!h->wstage_q.empty()) {
            CK(cudaMalloc(&h->d_weights_q, h->wstage_q.size()));
            CK(cudaMemcpy(h->d_weights_q, h->wstage_q.data(), h->wstage_q.size(), cudaMemcpyHostToDevice));
        }
        const size_t in_bytes = (size_t)Bm * Hn * Wn * 3;
        CK(cudaMalloc(&h->d_input, in_bytes));
        CK(cudaHostAlloc(&h->h_input, in_bytes, cudaHostAllocDefault));
        h->raw_bytes = ((size_t)h->cfg.max_image_w * h->cfg.max_image_h * 3 + 255) / 256 * 256;
        // one raw buffer per batch element (capped at 2 GiB in total): the images of a call are uploaded back to back and
        // letter-boxed by ONE launch
        h->raw_slots = (int)std::max<size_t>(1, std::min<size_t>((size_t)Bm, ((size_t)2 << 30) / h->raw_bytes));
        CK(cudaMalloc(&h->d_raw, h->raw_bytes * h->raw_slots));
        CK(cudaHostAlloc(&h->h_raw, 2 * h->raw_bytes, cudaHostAllocDefault));
        for (auto &e : h->raw_ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        CK(cudaHostAlloc(&h->h_dets, sizeof(rf_det) * (size_t)Bm * h->cfg.max_faces, cudaHostAllocDefault));
        CK(cudaHostAlloc(&h->h_counts, sizeof(int) * 2 * Bm, cudaHostAllocDefault));
        CK(cudaHostAlloc(&h->tile_dbg, 64, cudaHostAllocMapped));
        memset(h->tile_dbg, 0, 64);
        CK(cudaHostGetDevicePointer(&h->tile_dbg_dev, h->tile_dbg, 0));
        h->ctx.resize(h->cfg.streams <= 0 ? RF_MAX_STREAMS : std::min(h->cfg.streams, RF_MAX_STREAMS));
        for (Ctx &c : h->ctx) create_ctx(h, c, true);
        for (int l = 0; l < 3; l++) {
            const int ch[3] = {4, 8, 20};
            for (int k = 0; k < 3; k++) h->blob_elems[3 * l + k] = (size_t)ch[k] * h->lv[l].h * h->lv[l].w;
        }
        CK(cudaDeviceSynchronize());
    } catch (const CudaFail &f) {
        return fail_cuda(nullptr, f);
    } catch (const PlanFail &f) {
        return fail(nullptr, f.status, "rf_create: " + f.msg);
    }
    *out = H.release();
    return RF_OK;
}

void rf_destroy(rf_handle h) { destroy(h); }

uint8_t *rf_pinned_input(rf_handle h) { return h ? h->h_input : nullptr; }
uint8_t *rf_device_input(rf_handle h) { return h ? h->d_input : nullptr; }

int rf_get_net_size(rf_handle h, int *net_w, int *net_h, int *max_batch, int *max_faces) {
    if (!h) return RF_ERR_INVALID_ARG;
    if (net_w) *net_w = h->cfg.net_w;
    if (net_h) *net_h = h->cfg.net_h;
    if (max_batch) *max_batch = h->cfg.max_batch;
    if (max_faces) *max_faces = h->cfg.max_faces;
    return RF_OK;
}
int rf_num_anchors(rf_handle h) { return h ? h->ctx[0].pb.anchors_per_image : RF_ERR_INVALID_ARG; }
void *rf_stream(rf_handle h) { return h ? (void *)h->ctx[0].stream : nullptr; }

int rf_synchronize(rf_handle h) {
    if (!h) return RF_ERR_INVALID_ARG;
    try {
        CK(cudaSetDevice(h->device));
        for (Ctx &c : h->ctx) CK(cudaStreamSynchronize(c.stream));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// Orders context 0's stream (the one rf_stream returns) after everything queued so far on every context.
int rf_fence(rf_handle h) {
    if (!h) return RF_ERR_INVALID_ARG;
    try {
        CK(cudaSetDevice(h->device));
        for (size_t c = 1; c < h->ctx.size(); c++) {
            CK(cudaEventRecord(h->ctx[c].fence, h->ctx[c].stream));
            CK(cudaStreamWaitEvent(h->ctx[0].stream, h->ctx[c].fence, 0));
        }
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

void *rf_last_stream(rf_handle h) { return h ? (void *)(h->last_stream ? h->last_stream : h->ctx[0].stream) : nullptr; }

int rf_launches_per_batch(rf_handle h, int n) {
    (void)n;
    return h ? (int)h->steps.size() : RF_ERR_INVALID_ARG;
}

// `ran_on` (optional) receives the context the forward was issued on.  `stage` (optional) issues work on that context's stream
// ahead of the forward and returns the input tensor the forward reads instead of dev_bgr.
static int detect_device_impl(rf_handle h, const uint8_t *dev_bgr, int n, float thr, float nms, const rf_det **dev_dets, const int32_t **dev_counts,
                              bool gather, Ctx **ran_on = nullptr, const std::function<const uint8_t *(Ctx &)> &stage = nullptr) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (gather && (!h->comm.ready || n == 0)) return fail(h, RF_ERR_INVALID_ARG, "rf_detect_batch_device_allgather: call rf_comm_init first (and n > 0)");
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[h->next_dev_ctx++ % h->ctx.size()];   // consecutive batches overlap on different contexts
        if (ran_on) *ran_on = &c;
        h->last_stream = c.stream;
        // the caller's device images are read in place (conv0 takes the pointer from the run parameters)
        if (c.param_seq && c.param_seq % Ctx::kParamSlots == 0) CK(cudaStreamSynchronize(c.stream));
        if (stage) dev_bgr = stage(c);
        const unsigned seq = gather ? ++h->comm.seq : 0u;
        set_params(h, c, thr, nms, dev_bgr, seq);
        if (n > 0) forward_graph(h, c, n);
        const rf_det *dets = c.pb.out_dets;
        const int32_t *counts = c.pb.out_counts;
        if (gather) {
            const unsigned slot = seq % (unsigned)h->comm.ring;
            const size_t img0 = (size_t)slot * h->comm.world * h->cfg.max_batch;
            dets = c.pb.comm.dets[h->comm.rank] + img0 * h->cfg.max_faces;
            counts = c.pb.comm.counts[h->comm.rank] + img0;
        }
        if (dev_dets) *dev_dets = dets;
        if (dev_counts) *dev_counts = counts;
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_detect_batch_device(rf_handle h, const uint8_t *dev_bgr, int n, float thr, float nms, const rf_det **dev_dets,
                           const int32_t **dev_counts) {
    return detect_device_impl(h, dev_bgr, n, thr, nms, dev_dets, dev_counts, false);
}
int rf_detect_batch_device_allgather(rf_handle h, const uint8_t *dev_bgr, int n, float thr, float nms, const rf_det **all_dets,
                                     const int32_t **all_counts) {
    return detect_device_impl(h, dev_bgr, n, thr, nms, all_dets, all_counts, true);
}

// Kept records of images [first, first + n) -> the caller's arrays, image g at the same place on both sides (max_faces
// records per image).  Counts are clamped to max_faces: those of other ranks come from peer memory.
static void put_results(rf_handle h, const rf_det *dets, const int *counts, size_t first, int n, rf_face *out_faces, int *out_counts,
                        int32_t *out_idx) {
    const int mf = h->cfg.max_faces;
    for (size_t g = first; g < first + n; g++) {
        const int k = std::min(counts[g], mf);
        if (out_counts) out_counts[g] = k;
        for (int j = 0; j < k; j++) {
            const rf_det &d = dets[g * mf + j];
            if (out_faces) out_faces[g * mf + j] = d.face;
            if (out_idx) out_idx[g * mf + j] = d.anchor_index;
        }
    }
}

// Waits for the results of n images in pb (written on stream s) and copies them out (through the pinned h_counts / h_dets).
static void fetch_post(rf_handle h, const PostBuffers &pb, cudaStream_t s, int n, rf_face *out_faces, int *out_counts, int32_t *out_idx) {
    CK(cudaMemcpyAsync(h->h_counts, pb.out_counts, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(h->h_dets, pb.out_dets, sizeof(rf_det) * (size_t)n * h->cfg.max_faces, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    put_results(h, h->h_dets, h->h_counts, 0, n, out_faces, out_counts, out_idx);
}
static void fetch_results(rf_handle h, Ctx &c, int n, rf_face *out_faces, int *out_counts, int32_t *out_idx) {
    fetch_post(h, c.pb, c.stream, n, out_faces, out_counts, out_idx);
}

// Whether `p` is page-locked host memory (cudaHostAlloc / cudaHostRegister), which an H2D copy may read in place.
static bool is_pinned(const void *p) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost) return true;
    cudaGetLastError();
    return false;
}

// H2D copies of network-sized images i -> dst + i * img_bytes, issued on `s` in runs: consecutive images whose sources are
// adjacent in host memory go as one copy.
struct H2DRuns {
    uint8_t *dst;
    size_t img_bytes;
    cudaStream_t s;
    const uint8_t *src = nullptr;
    int start = -1, len = 0;
    void add(int i, const uint8_t *p) {
        if (start >= 0 && i == start + len && p == src + (size_t)len * img_bytes) { len++; return; }
        flush();
        start = i; src = p; len = 1;
    }
    void flush() {
        if (start >= 0) CK(cudaMemcpyAsync(dst + (size_t)start * img_bytes, src, (size_t)len * img_bytes, cudaMemcpyHostToDevice, s));
        start = -1;
    }
};

extern "C++" {
// One host plane of `rows` rows of row_bytes (pitch bytes apart) -> d_dst, packed, on `s`.  Pinned sources (cudaHostAlloc /
// cudaHostRegister) are copied straight from the caller's memory, row stride and all.  Pageable sources are staged through the
// two pinned buffers (each plane fits one: it is at most a max_image BGR image): a row-band parallel host copy (host_copy.h) into
// one buffer overlaps the DMA out of the other; the only host wait is for the DMA that last read the buffer about to be
// overwritten.  In both cases the stream orders the copy into d_raw behind the letter-box kernel that still reads the previous image.
void rf_eng::upload_plane(rf_handle h, cudaStream_t s, uint8_t *d_dst, const uint8_t *src, size_t row_bytes, size_t pitch, int rows) {
    if (is_pinned(src)) {
        CK(cudaMemcpy2DAsync(d_dst, row_bytes, src, pitch, row_bytes, (size_t)rows, cudaMemcpyHostToDevice, s));
        return;
    }
    if (!h->copy_pool) h->copy_pool.reset(new HostCopyPool((int)std::min(3u, std::max(1u, std::thread::hardware_concurrency()) - 1u)));
    const int slot = (int)(h->raw_seq++ & 1u);
    uint8_t *buf = h->h_raw + (size_t)slot * h->raw_bytes;
    CK(cudaEventSynchronize(h->raw_ev[slot]));      // (returns at once for an event never recorded)
    h->copy_pool->copy_rows(buf, src, row_bytes, pitch, rows);
    CK(cudaMemcpyAsync(d_dst, buf, row_bytes * rows, cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(h->raw_ev[slot], s));
}

int rf_eng::check_orientations(rf_handle h, const char *who, const int *orientations, int n) {
    if (n > 0 && !orientations) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: orientations is NULL", who));
    for (int i = 0; i < n; i++)
        if (lb_orientation_bits(orientations[i]) < 0)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: item %d: orientation %d, must be in 1..8 (EXIF)", who, i, orientations[i]));
    return RF_OK;
}

// Checks n, the matrix and every frame descriptor; nothing is launched before this passes.
int rf_eng::check_frames(rf_handle h, const char *who, const rf_yuv_frame *frames, int n, int matrix) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (n > 0 && !frames) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frames is NULL", who));
    if (matrix != RF_YUV_BT601 && matrix != RF_YUV_BT709) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: unknown matrix %d", who, matrix));
    for (int i = 0; i < n; i++) {
        const rf_yuv_frame &f = frames[i];
        if (f.width <= 0 || f.height <= 0 || (f.width & 1) || (f.height & 1))
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d is %dx%d; 4:2:0 sizes must be positive and even", who, i, f.width, f.height));
        if (!f.y || !f.u || !f.v) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d has a NULL plane", who, i));
        if (f.uv_step != 1 && f.uv_step != 2) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: uv_step %d, must be 1 or 2", who, i, f.uv_step));
        const uintptr_t u = (uintptr_t)f.u, v = (uintptr_t)f.v;
        if (f.uv_step == 2 && u != v + 1 && v != u + 1)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: semi-planar u and v must be adjacent bytes of one plane", who, i));
        if (f.y_pitch < f.width || f.uv_pitch < f.width / 2 * f.uv_step)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: pitches %d / %d below the row bytes %d / %d", who, i, f.y_pitch, f.uv_pitch, f.width,
                                                   f.width / 2 * f.uv_step));
        if (f.width > h->cfg.max_image_w || f.height > h->cfg.max_image_h)
            return fail(h, RF_ERR_CAPACITY, fmt("%s: frame %d is %dx%d, larger than max_image %dx%d", who, i, f.width, f.height, h->cfg.max_image_w,
                                                h->cfg.max_image_h));
    }
    return RF_OK;
}
}  // extern "C++"


extern "C++" {
// the displayed size of image i: its stored size, transposed for EXIF orientations 5..8
template <typename Source>
static void displayed_size(const Source &src, int i, int &w, int &hgt) {
    const bool t = (src.bits(i) & LB_TRANSPOSE) != 0;
    w = t ? src.height(i) : src.width(i);
    hgt = t ? src.width(i) : src.height(i);
}
}  // extern "C++"

// ---- f5 face alignment (align.cuh) ----------------------------------------------------------------------------------------------
extern "C++" {
// Checks the caller's rf_align_params and fills the image-independent kernel arguments (defaults applied).
int rf_eng::align_setup(rf_handle h, const char *who, const rf_align_params *p, AlignArgs &a) {
    if (!p) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: params is NULL", who));
    a = AlignArgs{};
    a.crop_w = p->crop_w; a.crop_h = p->crop_h;
    if (a.crop_w == 0 && a.crop_h == 0) a.crop_w = a.crop_h = 112;
    if (a.crop_w < ALIGN_MIN_SIDE || a.crop_w > ALIGN_MAX_SIDE || a.crop_h < ALIGN_MIN_SIDE || a.crop_h > ALIGN_MAX_SIDE)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: crop %dx%d, each side must be in [%d, %d]", who, p->crop_w, p->crop_h, ALIGN_MIN_SIDE, ALIGN_MAX_SIDE));
    if (p->format != RF_CROP_BGR_U8 && p->format != RF_CROP_RGB_F32 && p->format != RF_CROP_RGB_F16)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: unknown crop format %d", who, p->format));
    if (p->max_faces < 0 || p->max_faces > h->cfg.max_faces)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: max_faces %d, must be in [0, %d] (the handle's max_faces)", who, p->max_faces, h->cfg.max_faces));
    float mean = p->mean, sd = p->std;
    if (mean == 0.f && sd == 0.f) mean = sd = 127.5f;
    if (sd == 0.f || !std::isfinite(sd) || !std::isfinite(mean)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: std must be finite and non-zero", who));
    // insightface's arcface_dst: left eye, right eye, nose, left and right mouth corner in a 112 x 112 crop
    static const float arcface[10] = {38.2946f, 51.6963f, 73.5318f, 51.5014f, 56.0252f, 71.7366f, 41.5493f, 92.3655f, 70.7299f, 92.2041f};
    bool given = false;
    for (int k = 0; k < 10; k++) given |= p->template_xy[k] != 0.f;
    for (int k = 0; k < 10; k++) a.tmpl[k] = (double)(given ? p->template_xy[k] : arcface[k]);
    a.max_align = p->max_faces ? p->max_faces : h->cfg.max_faces;
    a.format = p->format;
    a.mean = mean;
    a.inv_std = (float)(1.0 / (double)sd);
    a.crop_bytes = align_crop_bytes(a.crop_w, a.crop_h, a.format);
    return RF_OK;
}


// The align checks of every entry point that crops: the params, somewhere for the crops to go and -- the blocking paths cut the
// crops from the originals after the forward -- a raw buffer of its own for each of the `resident` originals that need one.
int rf_eng::check_align(rf_handle h, const char *who, const rf_align_params *p, int n, const void *crops, int resident, AlignArgs &a) {
    int rc = align_setup(h, who, p, a);
    if (rc) return rc;
    if (n > 0 && !crops) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: align without a crop buffer", who));
    if (resident > h->raw_slots)
        return fail(h, RF_ERR_CAPACITY, fmt("%s: %d images need a raw buffer until their crops are cut, but the handle keeps at most %d "
                                            "originals resident (one %dx%d raw buffer each); split the batch", who, resident, h->raw_slots,
                                            h->cfg.max_image_w, h->cfg.max_image_h));
    return RF_OK;
}
}  // extern "C++"

// Makes room for n images' crops and the matrices of the blocking align paths (context 0).
static void ensure_align_buffers(rf_handle h, int n, const AlignArgs &a) {
    if (!h->d_align_mats) CK(cudaMalloc(&h->d_align_mats, sizeof(double) * 6 * h->cfg.max_batch * h->cfg.max_faces));
    const size_t need = (size_t)n * a.max_align * a.crop_bytes;
    if (need > h->align_crops_bytes) {
        CK(cudaFree(h->d_align_crops));
        h->d_align_crops = nullptr;
        h->align_crops_bytes = 0;
        CK(cudaMalloc(&h->d_align_crops, need));
        h->align_crops_bytes = need;
    }
}

// After fetch_results on context c: the kept faces of image i (h_dets) mapped back by scale(i), network-input pixels -> image
// pixels (k_merge_views' map-back), into out_faces; with `a`, the crops (and matrices) of its first min(count, A) faces copied
// out of the align buffers.  Blocking.
extern "C++" {
template <typename ScaleOf>
static void put_mapped(rf_handle h, Ctx &c, int n, ScaleOf scale, const AlignArgs *a, rf_face *out_faces, void *out_crops, double *out_mats) {
    const int mf = h->cfg.max_faces;
    for (int i = 0; i < n; i++) {
        const int k = h->h_counts[i];
        const float s = scale(i);
        for (int j = 0; out_faces && j < k; j++) {
            rf_face f = h->h_dets[(size_t)i * mf + j].face;
            f.x1 *= s; f.y1 *= s; f.x2 *= s; f.y2 *= s;
            for (int l = 0; l < 5; l++) { f.lx[l] *= s; f.ly[l] *= s; }
            out_faces[(size_t)i * mf + j] = f;
        }
        if (!a) continue;
        const size_t first = (size_t)i * a->max_align, m = (size_t)std::min(k, a->max_align);
        if (!m) continue;
        CK(cudaMemcpyAsync(static_cast<uint8_t *>(out_crops) + first * a->crop_bytes, static_cast<uint8_t *>(h->d_align_crops) + first * a->crop_bytes,
                           m * a->crop_bytes, cudaMemcpyDeviceToHost, c.stream));
        if (out_mats)
            CK(cudaMemcpyAsync(out_mats + first * 6, h->d_align_mats + first * 6, m * 6 * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
    }
    CK(cudaStreamSynchronize(c.stream));
}
}  // extern "C++"


// The blocking letter-box path of rf_detect_batch, rf_detect_align_batch, rf_detect_oriented_batch and rf_detect_yuv_batch, on
// context 0.  Network-sized packed upright images are copied H2D straight from the caller's memory when it is pinned
// (cudaHostAlloc / cudaHostRegister / the library's own rf_pinned_input), otherwise via the library's pinned mirror; runs of
// adjacent sources collapse into one copy.  Every other image is uploaded into a raw buffer of its own, a chunk of raw_slots at a
// time, each chunk letter-boxed by one launch (RF_FLAG_NPP_RESIZE: the reference's NPP super-sampling definition instead of its
// OpenCV bilinear one).  With `aligned`, the check has made sure that no raw buffer is recycled within the call, and the crops are
// cut from the originals after the forward.  `map_back`: faces in image pixels rather than network-input pixels.
extern "C++" {
template <typename Source>
static int detect_blocking(rf_handle h, const char *who, const Source &src, int n, float thr, float nms, bool aligned, const rf_align_params *align,
                           bool map_back, rf_face *out_faces, int *out_counts, int32_t *out_idx, void *out_crops, double *out_mats) {
    using Src = typename Source::Src;
    int rc = src.check(h, who, n);
    if (rc) return rc;
    AlignArgs a;
    if (aligned) {
        int raw = 0;
        for (int i = 0; i < n; i++) raw += !src.direct(h, i);
        if ((rc = check_align(h, who, align, n, out_crops, raw, a))) return rc;
    }
    if (n == 0) return RF_OK;
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
    const size_t img_bytes = (size_t)Hn * Wn * 3;
    const int area = (h->cfg.flags & RF_FLAG_NPP_RESIZE) ? 1 : 0;
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        if (aligned) ensure_align_buffers(h, n, a);
        // where each original stays resident, and its map-back factor (only the crops and the map-back read them)
        std::vector<AlignImageT<Src>> orig(aligned || map_back ? n : 0);
        H2DRuns runs{h->d_input, img_bytes, c.stream};
        bool staging_dirty = false;
        std::vector<LbItemT<Src>> lb;
        for (int i = 0; i < n; i++) {
            if constexpr (std::is_same<Src, BgrRows>::value) {
                if (src.direct(h, i)) {
                    const uint8_t *p = src.imgs[i];
                    const bool in_mirror = p >= h->h_input && p < h->h_input + (size_t)h->cfg.max_batch * img_bytes;
                    if (!in_mirror && !is_pinned(p)) {
                        if (!staging_dirty) { CK(cudaStreamSynchronize(c.stream)); staging_dirty = true; }
                        uint8_t *slot = h->h_input + (size_t)i * img_bytes;
                        memcpy(slot, p, img_bytes);
                        p = slot;
                    }
                    runs.add(i, p);
                    if (!orig.empty()) orig[i] = AlignImageT<Src>{BgrRows{h->d_input + (size_t)i * img_bytes, Wn * 3}, Wn, Hn, 1.f, 0};
                    continue;
                }
                runs.flush();
            }
            // a full chunk of raw buffers is letter-boxed before the next image reuses the first (stream order)
            if ((int)lb.size() == h->raw_slots) { CK(launch_letterbox_batch(lb.data(), (int)lb.size(), Wn, Hn, c.stream)); lb.clear(); }
            const Src p = src.upload(h, c.stream, i, (int)lb.size());
            const int bits = src.bits(i);
            int dw, dh;
            displayed_size(src, i, dw, dh);
            lb.emplace_back();
            const float scale = letterbox_fill(lb.back(), p, dw, dh, h->d_input + (size_t)i * img_bytes, Wn, Hn, bits, area);
            if (!orig.empty()) orig[i] = AlignImageT<Src>{p, dw, dh, scale, bits};
        }
        runs.flush();
        if (!lb.empty()) CK(launch_letterbox_batch(lb.data(), (int)lb.size(), Wn, Hn, c.stream));
        set_params(h, c, thr, nms);
        forward_graph(h, c, n);
        if (aligned) {
            a.n = n;
            a.crops = h->d_align_crops;
            a.mats = out_mats ? h->d_align_mats : nullptr;
            CK(launch_align_faces(a, orig.data(), c.pb, h->num_sms, c.stream, src.oriented));
        }
        fetch_results(h, c, n, map_back ? nullptr : out_faces, out_counts, out_idx);
        if (map_back) put_mapped(h, c, n, [&](int i) { return orig[i].scale; }, aligned ? &a : nullptr, out_faces, out_crops, out_mats);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}
}  // extern "C++"

int rf_detect_batch(rf_handle h, const uint8_t *const *imgs, const int *widths, const int *heights, const int *row_strides,
                    int n, float thr, float nms, rf_face *out_faces, int *out_counts, int32_t *out_idx) {
    return detect_blocking(h, "rf_detect_batch", BgrImages{imgs, widths, heights, row_strides, nullptr, false}, n, thr, nms, false, nullptr,
                           false, out_faces, out_counts, out_idx, nullptr, nullptr);
}

int rf_detect_align_batch(rf_handle h, const uint8_t *const *imgs, const int *widths, const int *heights, const int *row_strides,
                          int n, float thr, float nms, const rf_align_params *params, rf_face *out_faces, int *out_counts,
                          void *out_crops, double *out_mats) {
    return detect_blocking(h, "rf_detect_align_batch", BgrImages{imgs, widths, heights, row_strides, nullptr, false}, n, thr, nms, true, params,
                           true, out_faces, out_counts, nullptr, out_crops, out_mats);
}

// f9 oriented images (rf_b200.h rf_detect_oriented_batch)
int rf_detect_oriented_batch(rf_handle h, const uint8_t *const *imgs, const int *widths, const int *heights, const int *row_strides,
                             const int *orientations, int n, float thr, float nms, const rf_align_params *align, rf_face *out_faces,
                             int *out_counts, int32_t *out_idx, void *out_crops, double *out_mats) {
    return detect_blocking(h, "rf_detect_oriented_batch", BgrImages{imgs, widths, heights, row_strides, orientations, true}, n, thr, nms,
                           align != nullptr, align, true, out_faces, out_counts, out_idx, out_crops, out_mats);
}

// f6 video frames: YUV 4:2:0 (yuv.cuh)
int rf_detect_yuv_batch(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, float thr, float nms, const rf_align_params *align,
                        rf_face *out_faces, int *out_counts, int32_t *out_idx, void *out_crops, double *out_mats) {
    return detect_blocking(h, "rf_detect_yuv_batch", YuvFrames{frames, matrix, nullptr, false}, n, thr, nms, align != nullptr, align, true,
                           out_faces, out_counts, out_idx, out_crops, out_mats);
}

int rf_detect_align_batch_device(rf_handle h, const uint8_t *dev_bgr, int n, float thr, float nms, const rf_align_params *params,
                                 void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts) {
    if (!h) return RF_ERR_INVALID_ARG;
    AlignArgs a;
    int rc = check_align(h, "rf_detect_align_batch_device", params, n, dev_crops, 0, a);
    if (rc) return rc;
    Ctx *c = nullptr;
    if ((rc = detect_device_impl(h, dev_bgr, n, thr, nms, dev_dets, dev_counts, false, &c))) return rc;
    if (n == 0) return RF_OK;
    // the crops are cut from the network-sized images the forward read
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
    const uint8_t *base = dev_bgr ? dev_bgr : h->d_input;
    std::vector<AlignImageT<BgrRows>> table(n);
    for (int i = 0; i < n; i++) table[i] = AlignImageT<BgrRows>{BgrRows{base + (size_t)i * Hn * Wn * 3, Wn * 3}, Wn, Hn, 1.f, 0};
    a.n = n;
    a.crops = dev_crops;
    a.mats = dev_mats;
    try {
        CK(launch_align_faces(a, table.data(), c->pb, h->num_sms, c->stream));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

extern "C++" {
// rf_detect_yuv_batch_device, rf_detect_yuv_oriented_device and the detect half of rf_detect_yuv_track_device: the frames are
// letter-boxed on the context the forward lands on, into that context's own input tensor, and cropped in place.
int rf_eng::yuv_device_impl(rf_handle h, const char *who, const YuvFrames &src, int n, float thr, float nms, const rf_align_params *align,
                            void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    int rc = src.check(h, who, n);
    if (rc) return rc;
    AlignArgs a;
    if (align && (rc = check_align(h, who, align, n, dev_crops, 0, a))) return rc;
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
    const size_t img_bytes = (size_t)Hn * Wn * 3;
    const int area = (h->cfg.flags & RF_FLAG_NPP_RESIZE) ? 1 : 0;
    std::vector<AlignImageT<YuvPlanes>> orig(n);
    auto stage = [&](Ctx &c) -> const uint8_t * {
        if (!c.d_frames_in) CK(cudaMalloc(&c.d_frames_in, (size_t)h->cfg.max_batch * img_bytes));
        std::vector<LbYuvItem> lb(n);
        for (int i = 0; i < n; i++) {
            const YuvPlanes p = src.in_place(i);
            const int bits = src.bits(i);
            int dw, dh;
            displayed_size(src, i, dw, dh);
            orig[i] = AlignImageT<YuvPlanes>{p, dw, dh, letterbox_fill(lb[i], p, dw, dh, c.d_frames_in + i * img_bytes, Wn, Hn, bits, area), bits};
            if (out_scales) out_scales[i] = orig[i].scale;
        }
        CK(launch_letterbox_batch(lb.data(), n, Wn, Hn, c.stream));
        return c.d_frames_in;
    };
    Ctx *c = nullptr;
    if ((rc = detect_device_impl(h, nullptr, n, thr, nms, dev_dets, dev_counts, false, &c, stage))) return rc;
    if (n == 0 || !align) return RF_OK;
    a.n = n;
    a.crops = dev_crops;
    a.mats = dev_mats;
    try {
        CK(launch_align_faces(a, orig.data(), c->pb, h->num_sms, c->stream, src.oriented));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}
}  // extern "C++"

int rf_detect_yuv_batch_device(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, float thr, float nms, const rf_align_params *align,
                               void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    return yuv_device_impl(h, "rf_detect_yuv_batch_device", YuvFrames{frames, matrix, nullptr, false}, n, thr, nms, align, dev_crops, dev_mats,
                           dev_dets, dev_counts, out_scales);
}

int rf_detect_yuv_oriented_device(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n, int matrix, float thr, float nms,
                                  const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                                  const int32_t **dev_counts, float *out_scales) {
    return yuv_device_impl(h, "rf_detect_yuv_oriented_device", YuvFrames{frames, matrix, orientations, true}, n, thr, nms, align, dev_crops,
                           dev_mats, dev_dets, dev_counts, out_scales);
}

// ---- f7 tiled detection: a scale pyramid cut into network-sized tiles (preprocess.cuh tile_layout) ----------------------------------
int rf_tile_layout(int net_w, int net_h, int width, int height, const rf_tiling *t, rf_tile *out, int cap) {
    if (cap < 0 || (cap > 0 && !out)) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_tile_layout: cap < 0 or out is NULL");
    std::vector<rf_tile> tiles;
    std::string err;
    const int rc = tile_layout(net_w, net_h, width, height, t, tiles, &err);
    if (rc) return fail(nullptr, rc, "rf_tile_layout: " + err);
    std::copy_n(tiles.begin(), std::min<size_t>(tiles.size(), (size_t)cap), out);
    return (int)tiles.size();
}


extern "C++" {
// Whether the handle can tile: levels are cv::resize's, so not with the NPP resize definition.
int rf_eng::tiling_supported(rf_handle h, const char *who) {
    if (h->cfg.flags & RF_FLAG_NPP_RESIZE)
        return fail(h, RF_ERR_UNSUPPORTED, fmt("%s: tiles are levels of cv::resize; the handle letter-boxes with NPPI_INTER_SUPER, which "
                                               "only down-samples", who));
    return RF_OK;
}

// The checks every tiled path shares, after its source check: the resize definition and each image's layout, of its displayed size
// (f21: an oriented image is tiled as the displayed image D = T_o(S)).
template <typename Source>
static int tiled_layouts(rf_handle h, const char *who, const Source &src, int n, const rf_tiling *t, std::vector<std::vector<rf_tile>> &layouts) {
    if (int rc = tiling_supported(h, who)) return rc;
    layouts.resize(n);
    for (int i = 0; i < n; i++) {
        std::string err;
        int dw, dh;
        displayed_size(src, i, dw, dh);
        const int rc = tile_layout(h->cfg.net_w, h->cfg.net_h, dw, dh, t, layouts[i], &err);
        if (rc) return fail(h, rc, fmt("%s: image %d: %s", who, i, err.c_str()));
    }
    return RF_OK;
}

// The front end of every tiled entry point: the source check, the layouts, then the align checks (`resident`: the blocking paths
// keep every original in a raw buffer of its own until the crops are cut).
template <typename Source>
static int tiled_check(rf_handle h, const char *who, const Source &src, int n, const rf_tiling *t, bool aligned, const rf_align_params *align,
                       const void *crops, bool resident, std::vector<std::vector<rf_tile>> &layouts, AlignArgs &a) {
    int rc = src.check(h, who, n);
    if (rc) return rc;
    if ((rc = tiled_layouts(h, who, src, n, t, layouts))) return rc;
    return aligned ? check_align(h, who, align, n, crops, resident ? n : 0, a) : RF_OK;
}

// The network inputs of one chunk: letter-box items with their merge sources in batch slots 0 .. lb.size() - 1 (launch_merge reads
// contiguous slots from 0), then f24's warp views with their rotated merge sources in the slots after them.
template <typename Src>
struct ChunkWork {
    std::vector<LbItemT<Src>> lb;
    std::vector<MergeSource> ms;
    std::vector<WarpItemT<Src>> wp;
    std::vector<int> wp_bits;          // f25: each warp item's LB_* orientation bits (0: an upright frame)
    std::vector<RotatedSource> rs;
};
// One network input of a chunked call: tile `item` of image `image`'s layout, or view `item` of it (f24).
struct Job { int image, item; };

// The jobs of the tiled paths: every tile of each image's layout.
template <typename Source>
struct TileJobs {
    rf_handle h;
    const Source &source;
    const std::vector<std::vector<rf_tile>> &layouts;
    int count(int i) const { return (int)layouts[i].size(); }
    void fill(const Job *jobs, int m, const std::vector<typename Source::Src> &src, uint8_t *input, ChunkWork<typename Source::Src> &w) const {
        const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
        const size_t img_bytes = (size_t)Hn * Wn * 3;
        w.lb.resize(m);
        w.ms.resize(m);
        for (int b = 0; b < m; b++) {
            const Job r = jobs[b];
            const rf_tile &tl = layouts[r.image][r.item];
            int dw, dh;
            displayed_size(source, r.image, dw, dh);
            tile_fill(w.lb[b], src[r.image], dw, dh, source.bits(r.image), input + b * img_bytes, Wn, Hn, tl);
            // records stay in displayed pixels: a mirrored level is un-mirrored with the displayed width (k_merge<false>)
            w.ms[b] = tile_source(r.image, r.item, h->cfg.max_faces, tl, dw);
        }
    }
};

// Chunked detection of n checked images, into `dst` (its candidate lists empty: allocation and every k_nms leave them so), the final
// NMS on `home`.  Image i contributes jobs.count(i) network inputs (tiles, or f24's views), which jobs.fill turns into a chunk's
// letter-box / warp items and merge sources.  The blocking paths upload image i into raw buffer `slot` on home, a `group` of raw
// buffers at a time; with `in_place` (one group), the device paths read the caller's memory.  The network inputs are made, detected
// and merged in chunks of up to max_batch, each chunk on the next context of the rf_detect_batch_device rotation, into that context's
// own input tensor.  Another context waits for `ready` -- recorded on home once the group's sources are on the device and `dst` may be
// written -- before its first letter-box of the group, or, with `in_place` (the sources are the caller's device memory), only before
// its first merge.  Home waits for every context the group used before the next group overwrites the raw buffers, and before the
// final NMS.
template <typename Source, typename Jobs>
static void detect_chunked(rf_handle h, const Source &source, int n, const Jobs &jobs, int group, bool in_place, Ctx &home, cudaEvent_t ready,
                           PostBuffers &dst, float thr, float nms, std::vector<typename Source::Src> &src) {
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w, B = h->cfg.max_batch;
    const size_t img_bytes = (size_t)Hn * Wn * 3;
    src.resize(n);
    for (int g0 = 0; g0 < n; g0 += group) {
        const int g1 = std::min(n, g0 + group);
        for (int i = g0; i < g1; i++) src[i] = in_place ? source.in_place(i) : source.upload(h, home.stream, i, i - g0);
        CK(cudaEventRecord(ready, home.stream));
        std::vector<Job> refs;
        for (int i = g0; i < g1; i++)
            for (int k = 0; k < jobs.count(i); k++) refs.push_back(Job{i, k});
        std::vector<char> joined(h->ctx.size(), 0);
        for (size_t k0 = 0; k0 < refs.size(); k0 += B) {
            const int m = (int)std::min<size_t>(B, refs.size() - k0);
            const size_t ci = h->next_dev_ctx++ % h->ctx.size();
            Ctx &c = h->ctx[ci];
            const bool wait = &c != &home && !joined[ci];
            if (wait && !in_place) CK(cudaStreamWaitEvent(c.stream, ready, 0));
            joined[ci] = 1;
            if (!c.d_frames_in) CK(cudaMalloc(&c.d_frames_in, (size_t)B * img_bytes));
            if (c.param_seq && c.param_seq % Ctx::kParamSlots == 0) CK(cudaStreamSynchronize(c.stream));
            ChunkWork<typename Source::Src> w;
            jobs.fill(&refs[k0], m, src, c.d_frames_in, w);
            CK(launch_letterbox_batch(w.lb.data(), (int)w.lb.size(), Wn, Hn, c.stream));
            CK(launch_letterbox_warp(w.wp.data(), (int)w.wp.size(), Wn, Hn, c.stream, w.wp_bits.data()));
            set_params(h, c, thr, nms, c.d_frames_in);
            forward_graph(h, c, m);
            if (wait && in_place) CK(cudaStreamWaitEvent(c.stream, ready, 0));
            CK(launch_merge(c.pb, w.ms.data(), (int)w.ms.size(), Wn, Hn, dst, c.stream));
            CK(launch_merge_rotated(c.pb, w.rs.data(), (int)w.rs.size(), dst, c.stream));
        }
        for (size_t ci = 0; ci < h->ctx.size(); ci++) {
            if (!joined[ci] || &h->ctx[ci] == &home) continue;
            CK(cudaEventRecord(h->ctx[ci].fence, h->ctx[ci].stream));
            CK(cudaStreamWaitEvent(home.stream, h->ctx[ci].fence, 0));
        }
    }
    // the final NMS over each image's candidates from all its network inputs reads its threshold from home's parameters
    if (home.param_seq && home.param_seq % Ctx::kParamSlots == 0) CK(cudaStreamSynchronize(home.stream));
    set_params(h, home, thr, nms);
    CK(launch_nms(n, home.d_params, dst, home.stream));
    CK(cudaGetLastError());
}

// The most network inputs any of the n images contributes: every one may contribute max_faces candidates.
template <typename Jobs>
static size_t most_jobs(const Jobs &jobs, int n) {
    int most = 0;
    for (int i = 0; i < n; i++) most = std::max(most, jobs.count(i));
    return (size_t)most;
}

// Makes room in pb for `most` * max_faces candidates per image.
static bool chunked_grow(rf_handle h, PostBuffers &pb, size_t most) {
    const int mf = h->cfg.max_faces;
    if ((size_t)pb.anchors_per_image >= most * mf) return false;
    free_post_buffers(pb);
    alloc_post_buffers(pb, (int)(most * mf), h->cfg.max_batch, mf);
    return true;
}


// The crops of every kept face in pb (a.crops / a.mats set by the caller), cut on s from the originals srcs at map-back factor 1
// (the merged records are in displayed image pixels; an oriented source reads its stored pixels through f9's oriented table).
template <typename Source>
static void tiled_crops(rf_handle h, AlignArgs a, int n, const Source &source, const std::vector<typename Source::Src> &srcs, const PostBuffers &pb,
                        cudaStream_t s) {
    std::vector<AlignImageT<typename Source::Src>> table(n);
    for (int i = 0; i < n; i++) {
        int dw, dh;
        displayed_size(source, i, dw, dh);
        table[i] = AlignImageT<typename Source::Src>{srcs[i], dw, dh, 1.f, source.bits(i)};
    }
    a.n = n;
    CK(launch_align_faces(a, table.data(), pb, h->num_sms, s, source.oriented));
}

// The blocking tiled paths: sources uploaded on context 0, merged into pb_tiles, fetched.  With `aligned`, the crops are cut on
// context 0 after the NMS and copied out with the faces.
template <typename Source>
static int detect_tiled_blocking(rf_handle h, const char *who, const Source &source, int n, const rf_tiling *t, float thr, float nms, bool aligned,
                                 const rf_align_params *align, rf_face *out_faces, int *out_counts, int32_t *out_tile_of, void *out_crops,
                                 double *out_mats) {
    std::vector<std::vector<rf_tile>> layouts;
    AlignArgs a;
    int rc = tiled_check(h, who, source, n, t, aligned, align, out_crops, true, layouts, a);
    if (rc || n == 0) return rc;
    try {
        CK(cudaSetDevice(h->device));
        const int mf = h->cfg.max_faces;
        const TileJobs<Source> jobs{h, source, layouts};
        chunked_grow(h, h->pb_tiles, most_jobs(jobs, n));
        Ctx &c0 = h->ctx[0];
        std::vector<typename Source::Src> srcs;
        detect_chunked(h, source, n, jobs, h->raw_slots, false, c0, c0.fence, h->pb_tiles, thr, nms, srcs);
        if (aligned) {
            ensure_align_buffers(h, n, a);
            a.crops = h->d_align_crops;
            a.mats = out_mats ? h->d_align_mats : nullptr;
            tiled_crops(h, a, n, source, srcs, h->pb_tiles, c0.stream);
        }
        fetch_post(h, h->pb_tiles, c0.stream, n, out_faces, out_counts, out_tile_of);
        if (out_tile_of)      // candidate id = tile * max_faces + rank
            for (int i = 0; i < n; i++)
                for (int j = 0; j < std::min(h->h_counts[i], mf); j++) out_tile_of[(size_t)i * mf + j] /= mf;
        if (aligned) put_mapped(h, c0, n, [](int) { return 1.f; }, &a, nullptr, out_crops, out_mats);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// The asynchronous chunked paths (tiles, and f24's rotated views): the caller's device sources src[i] read in place, merged into the
// next slot of `ring` (the tiled and the rotated calls each have their own), the final NMS and the crops on the home stream (the
// context the call's first chunk lands on), which rf_last_stream returns.
//   1. Home waits for the slot's `free` event before anything merges into it and records `start`; every other context waits for
//      `start` before its first merge (k_nms left the slot's candidate counts at zero).
//   2. A slot that must grow is freed only after the host has waited for `free`, and its counts are cleared on home before `start`.
//   3. Home joins every context it used through their fence events before the NMS.
//   4. The crops are cut on home after the NMS; then `free` is recorded.
//   5. A caller that reads the records later on home (a tracker call, f19) gets `free` back and records it again after its last read,
//      so that a later call on this slot, whose home may be another context, waits for those reads too.
// device_issue issues a checked call of n > 0 images (align: a.crops / a.mats set, or NULL; `free` may be NULL).
template <typename Source, typename Jobs>
static void device_issue(rf_handle h, std::vector<rf_handle_s::TiledSlot> &ring, unsigned &next_slot, const Source &source, int n,
                         const Jobs &jobs, float thr, float nms, const AlignArgs *align, const rf_det **dev_dets, const int32_t **dev_counts,
                         cudaEvent_t *free) {
    CK(cudaSetDevice(h->device));
    if (ring.empty()) {
        ring.resize(h->ctx.size());
        for (auto &s : ring) {
            CK(cudaEventCreateWithFlags(&s.free, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&s.start, cudaEventDisableTiming));
        }
    }
    rf_handle_s::TiledSlot &slot = ring[next_slot++ % ring.size()];
    Ctx &home = h->ctx[h->next_dev_ctx % h->ctx.size()];
    const size_t most = most_jobs(jobs, n);
    if ((size_t)slot.pb.anchors_per_image < most * h->cfg.max_faces) {
        CK(cudaEventSynchronize(slot.free));     // the slot's last call has finished with the buffers about to be freed
        chunked_grow(h, slot.pb, most);
        // alloc_post_buffers clears the counts on the legacy stream, which the contexts' streams do not wait for
        CK(cudaMemsetAsync(slot.pb.cand_count, 0, sizeof(int) * slot.pb.max_batch, home.stream));
    }
    CK(cudaStreamWaitEvent(home.stream, slot.free, 0));
    std::vector<typename Source::Src> srcs;
    detect_chunked(h, source, n, jobs, n, true, home, slot.start, slot.pb, thr, nms, srcs);
    if (align) tiled_crops(h, *align, n, source, srcs, slot.pb, home.stream);
    CK(cudaEventRecord(slot.free, home.stream));
    h->last_stream = home.stream;
    if (dev_dets) *dev_dets = slot.pb.out_dets;
    if (dev_counts) *dev_counts = slot.pb.out_counts;
    if (free) *free = slot.free;
}

template <typename Source>
static int detect_tiled_device(rf_handle h, const char *who, const Source &source, int n, const rf_tiling *t, float thr, float nms,
                               const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts) {
    std::vector<std::vector<rf_tile>> layouts;
    AlignArgs a;
    int rc = tiled_check(h, who, source, n, t, align != nullptr, align, dev_crops, false, layouts, a);
    if (rc || n == 0) return rc;
    a.crops = dev_crops;
    a.mats = dev_mats;
    try {
        device_issue(h, h->tiled_slots, h->next_tiled_slot, source, n, TileJobs<Source>{h, source, layouts}, thr, nms, align ? &a : nullptr,
                     dev_dets, dev_counts, nullptr);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// rf_detect_yuv_tiled_device's check and issue without crops, for the tracker's detect calls (tracker.cu).
int rf_eng::yuv_tiled_check(rf_handle h, const char *who, const YuvFrames &src, int n, const rf_tiling *t,
                            std::vector<std::vector<rf_tile>> &layouts) {
    AlignArgs a;
    return tiled_check(h, who, src, n, t, false, nullptr, nullptr, false, layouts, a);
}

int rf_eng::yuv_tiled_issue(rf_handle h, const YuvFrames &src, int n, const std::vector<std::vector<rf_tile>> &layouts, float thr, float nms,
                            const rf_det **dev_dets, const int32_t **dev_counts, cudaEvent_t *free) {
    try {
        device_issue(h, h->tiled_slots, h->next_tiled_slot, src, n, TileJobs<YuvFrames>{h, src, layouts}, thr, nms, nullptr, dev_dets,
                     dev_counts, free);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

}  // extern "C++"

int rf_detect_tiled(rf_handle h, const uint8_t *const *imgs, const int *widths, const int *heights, const int *row_strides, int n,
                    const rf_tiling *t, float thr, float nms, rf_face *out_faces, int *out_counts, int32_t *out_tile_of) {
    return detect_tiled_blocking(h, "rf_detect_tiled", BgrImages{imgs, widths, heights, row_strides, nullptr, false}, n, t, thr, nms, false,
                                 nullptr, out_faces, out_counts, out_tile_of, nullptr, nullptr);
}

int rf_detect_yuv_tiled(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_tiling *t, float thr, float nms,
                        rf_face *out_faces, int *out_counts, int32_t *out_tile_of) {
    return detect_tiled_blocking(h, "rf_detect_yuv_tiled", YuvFrames{frames, matrix, nullptr, false}, n, t, thr, nms, false, nullptr, out_faces,
                                 out_counts, out_tile_of, nullptr, nullptr);
}

int rf_detect_tiled_align(rf_handle h, const uint8_t *const *imgs, const int *widths, const int *heights, const int *row_strides, int n,
                          const rf_tiling *t, float thr, float nms, const rf_align_params *align, rf_face *out_faces, int *out_counts,
                          int32_t *out_tile_of, void *out_crops, double *out_mats) {
    return detect_tiled_blocking(h, "rf_detect_tiled_align", BgrImages{imgs, widths, heights, row_strides, nullptr, false}, n, t, thr, nms, true,
                                 align, out_faces, out_counts, out_tile_of, out_crops, out_mats);
}

int rf_detect_yuv_tiled_align(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_tiling *t, float thr, float nms,
                              const rf_align_params *align, rf_face *out_faces, int *out_counts, int32_t *out_tile_of, void *out_crops,
                              double *out_mats) {
    return detect_tiled_blocking(h, "rf_detect_yuv_tiled_align", YuvFrames{frames, matrix, nullptr, false}, n, t, thr, nms, true, align, out_faces,
                                 out_counts, out_tile_of, out_crops, out_mats);
}

int rf_detect_tiled_device(rf_handle h, const uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides, int n,
                           const rf_tiling *t, float thr, float nms, const rf_align_params *align, void *dev_crops, double *dev_mats,
                           const rf_det **dev_dets, const int32_t **dev_counts) {
    return detect_tiled_device(h, "rf_detect_tiled_device", BgrImages{dev_bgr, widths, heights, row_strides, nullptr, false}, n, t, thr, nms,
                               align, dev_crops, dev_mats, dev_dets, dev_counts);
}

int rf_detect_yuv_tiled_device(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_tiling *t, float thr, float nms,
                               const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                               const int32_t **dev_counts) {
    return detect_tiled_device(h, "rf_detect_yuv_tiled_device", YuvFrames{frames, matrix, nullptr, false}, n, t, thr, nms, align, dev_crops,
                               dev_mats, dev_dets, dev_counts);
}

// f21 oriented tiled detection (rf_b200.h): the tiled paths on the displayed images, through the same checks and issue
int rf_detect_tiled_oriented(rf_handle h, const uint8_t *const *imgs, const int *widths, const int *heights, const int *row_strides,
                             const int *orientations, int n, const rf_tiling *t, float thr, float nms, const rf_align_params *align,
                             rf_face *out_faces, int *out_counts, int32_t *out_tile_of, void *out_crops, double *out_mats) {
    return detect_tiled_blocking(h, "rf_detect_tiled_oriented", BgrImages{imgs, widths, heights, row_strides, orientations, true}, n, t, thr,
                                 nms, align != nullptr, align, out_faces, out_counts, out_tile_of, out_crops, out_mats);
}

int rf_detect_tiled_oriented_device(rf_handle h, const uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides,
                                    const int *orientations, int n, const rf_tiling *t, float thr, float nms, const rf_align_params *align,
                                    void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts) {
    return detect_tiled_device(h, "rf_detect_tiled_oriented_device", BgrImages{dev_bgr, widths, heights, row_strides, orientations, true}, n, t,
                               thr, nms, align, dev_crops, dev_mats, dev_dets, dev_counts);
}

int rf_detect_yuv_tiled_oriented_device(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n, int matrix, const rf_tiling *t,
                                        float thr, float nms, const rf_align_params *align, void *dev_crops, double *dev_mats,
                                        const rf_det **dev_dets, const int32_t **dev_counts) {
    return detect_tiled_device(h, "rf_detect_yuv_tiled_oriented_device", YuvFrames{frames, matrix, orientations, true}, n, t, thr, nms, align,
                               dev_crops, dev_mats, dev_dets, dev_counts);
}

// ---- parity hooks: the network input of one image ---------------------------------------------------------------------------------
// Image 0 of src uploaded into raw buffer 0 and letter-boxed (with `tiled`, tile `tile` of its layout) into `out`.
extern "C++" {
template <typename Source>
static int preprocess_one(rf_handle h, const char *who, const Source &src, bool tiled, const rf_tiling *t, int tile, uint8_t *out) {
    if (!h) return RF_ERR_INVALID_ARG;
    if (!out) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out is NULL", who));
    int rc = src.check(h, who, 1);
    if (rc) return rc;
    std::vector<std::vector<rf_tile>> layouts;
    if (tiled && (rc = tiled_layouts(h, who, src, 1, t, layouts))) return rc;
    if (tiled && (tile < 0 || tile >= (int)layouts[0].size()))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: tile %d, the layout has %zu", who, tile, layouts[0].size()));
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
    try {
        CK(cudaSetDevice(h->device));
        cudaStream_t s = h->ctx[0].stream;
        const typename Source::Src p = src.upload(h, s, 0, 0);
        LbItemT<typename Source::Src> it;
        int dw, dh;
        displayed_size(src, 0, dw, dh);
        if (tiled) tile_fill(it, p, dw, dh, src.bits(0), h->d_input, Wn, Hn, layouts[0][tile]);
        else letterbox_fill(it, p, dw, dh, h->d_input, Wn, Hn, src.bits(0), (h->cfg.flags & RF_FLAG_NPP_RESIZE) ? 1 : 0);
        CK(launch_letterbox_batch(&it, 1, Wn, Hn, s));
        CK(cudaMemcpyAsync(h->h_input, h->d_input, (size_t)Hn * Wn * 3, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        memcpy(out, h->h_input, (size_t)Hn * Wn * 3);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}
}  // extern "C++"

int rf_preprocess(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess", BgrImages{&bgr, &width, &height, &row_stride, nullptr, false}, false, nullptr, 0, out);
}
int rf_preprocess_oriented(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, int orientation, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_oriented", BgrImages{&bgr, &width, &height, &row_stride, &orientation, true}, false, nullptr, 0, out);
}
int rf_preprocess_yuv(rf_handle h, const rf_yuv_frame *frame, int matrix, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_yuv", YuvFrames{frame, matrix, nullptr, false}, false, nullptr, 0, out);
}
int rf_preprocess_yuv_oriented(rf_handle h, const rf_yuv_frame *frame, int matrix, int orientation, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_yuv_oriented", YuvFrames{frame, matrix, &orientation, true}, false, nullptr, 0, out);
}
int rf_preprocess_tile(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_tiling *t, int tile, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_tile", BgrImages{&bgr, &width, &height, &row_stride, nullptr, false}, true, t, tile, out);
}
int rf_preprocess_yuv_tile(rf_handle h, const rf_yuv_frame *frame, int matrix, const rf_tiling *t, int tile, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_yuv_tile", YuvFrames{frame, matrix, nullptr, false}, true, t, tile, out);
}
int rf_preprocess_tile_oriented(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, int orientation, const rf_tiling *t,
                                int tile, uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_tile_oriented", BgrImages{&bgr, &width, &height, &row_stride, &orientation, true}, true, t, tile, out);
}
int rf_preprocess_yuv_tile_oriented(rf_handle h, const rf_yuv_frame *frame, int matrix, int orientation, const rf_tiling *t, int tile,
                                    uint8_t *out) {
    return preprocess_one(h, "rf_preprocess_yuv_tile_oriented", YuvFrames{frame, matrix, &orientation, true}, true, t, tile, out);
}

// ---- f1 ingest: compressed images (main.cpp:18-26 decodes on the host with cv::imread) ---------------------------------------
int rf_detect_jpeg_batch(rf_handle h, const uint8_t *const *jpegs, const size_t *jpeg_bytes, int n, float thr, float nms, rf_face *out_faces,
                         int *out_counts, int32_t *out_idx, int *out_widths, int *out_heights) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (n == 0) return RF_OK;
    if (!jpegs || !jpeg_bytes) return fail(h, RF_ERR_INVALID_ARG, "rf_detect_jpeg_batch: NULL stream arrays");
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
    const size_t img_bytes = (size_t)Hn * Wn * 3;
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        std::vector<int> w(n), hg(n);
        for (int i = 0; i < n; i++) {
            if (!jpegs[i] || !jpeg_bytes[i]) return fail(h, RF_ERR_INVALID_ARG, fmt("rf_detect_jpeg_batch: stream %d is empty", i));
            if ((rc = jpeg_info(h, jpegs[i], jpeg_bytes[i], &w[i], &hg[i]))) return rc;
            if (w[i] <= 0 || hg[i] <= 0 || w[i] > h->cfg.max_image_w || hg[i] > h->cfg.max_image_h)
                return fail(h, RF_ERR_CAPACITY, fmt("JPEG %d is %dx%d, larger than max_image %dx%d", i, w[i], hg[i], h->cfg.max_image_w, h->cfg.max_image_h));
            if (out_widths) out_widths[i] = w[i];
            if (out_heights) out_heights[i] = hg[i];
        }
        const int area = (h->cfg.flags & RF_FLAG_NPP_RESIZE) ? 1 : 0;
        // network-sized images decode straight into the input tensor; the others into the raw buffers, a chunk of raw_slots at
        // a time, each chunk letter-boxed by one launch (all of it stream-ordered: a raw buffer is reused only behind its reader)
        for (int i0 = 0; i0 < n;) {
            std::vector<uint8_t *> dst;
            std::vector<LbItem> lb;
            int i1 = i0, used = 0;
            for (; i1 < n; i1++) {
                const bool direct = w[i1] == Wn && hg[i1] == Hn;
                if (!direct && used == h->raw_slots) break;
                dst.push_back(direct ? h->d_input + (size_t)i1 * img_bytes : h->d_raw + (size_t)used * h->raw_bytes);
                if (!direct) {
                    lb.emplace_back();
                    letterbox_fill(lb.back(), BgrRows{dst.back(), w[i1] * 3}, w[i1], hg[i1], h->d_input + (size_t)i1 * img_bytes, Wn, Hn, 0, area);
                    used++;
                }
            }
            if ((rc = jpeg_decode(h, jpegs + i0, jpeg_bytes + i0, i1 - i0, dst.data(), w.data() + i0, hg.data() + i0, c.stream))) return rc;
            if (!lb.empty()) CK(launch_letterbox_batch(lb.data(), (int)lb.size(), Wn, Hn, c.stream));
            i0 = i1;
        }
        set_params(h, c, thr, nms);
        forward_graph(h, c, n);
        fetch_results(h, c, n, out_faces, out_counts, out_idx);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_decode_jpeg(rf_handle h, const uint8_t *jpeg, size_t bytes, uint8_t *out_bgr, size_t out_capacity, int *width, int *height) {
    if (!h) return RF_ERR_INVALID_ARG;
    if (!jpeg || !bytes || !width || !height) return fail(h, RF_ERR_INVALID_ARG, "rf_decode_jpeg: NULL argument");
    try {
        CK(cudaSetDevice(h->device));
        cudaStream_t s = h->ctx[0].stream;
        int rc = jpeg_info(h, jpeg, bytes, width, height);
        if (rc) return rc;
        if (!out_bgr) return RF_OK;                                    // size query
        const size_t need = (size_t)*width * *height * 3;
        if (need > out_capacity) return fail(h, RF_ERR_CAPACITY, fmt("rf_decode_jpeg: %dx%d needs %zu bytes, the buffer has %zu", *width, *height, need, out_capacity));
        if (*width > h->cfg.max_image_w || *height > h->cfg.max_image_h)
            return fail(h, RF_ERR_CAPACITY, fmt("JPEG is %dx%d, larger than max_image %dx%d", *width, *height, h->cfg.max_image_w, h->cfg.max_image_h));
        uint8_t *dst = h->d_raw;
        if ((rc = jpeg_decode(h, &jpeg, &bytes, 1, &dst, width, height, s))) return rc;
        CK(cudaMemcpyAsync(out_bgr, h->d_raw, need, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

const char *rf_jpeg_backend(rf_handle h) { return h ? jpeg_backend(h) : "none"; }

static void ensure_slots(rf_handle h) {
    if (h->copy_stream) return;
    const size_t in_bytes = (size_t)h->cfg.max_batch * h->cfg.net_h * h->cfg.net_w * 3;
    CK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (auto &sl : h->slots) {
        CK(cudaMalloc(&sl.d_in, in_bytes));
        CK(cudaHostAlloc(&sl.h_in, in_bytes, cudaHostAllocDefault));
        CK(cudaHostAlloc(&sl.h_dets, sizeof(rf_det) * (size_t)h->cfg.max_batch * h->cfg.max_faces, cudaHostAllocDefault));
        CK(cudaHostAlloc(&sl.h_counts, sizeof(int) * h->cfg.max_batch, cudaHostAllocDefault));
        CK(cudaEventCreateWithFlags(&sl.ev_h2d, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming));
    }
}

static int submit_impl(rf_handle h, const uint8_t *const *imgs, int n, float thr, float nms, int *ticket, bool gather) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (!imgs || !ticket || n == 0) return fail(h, RF_ERR_INVALID_ARG, "rf_submit_batch: NULL argument or empty batch");
    if (gather && !h->comm.ready) return fail(h, RF_ERR_INVALID_ARG, "rf_submit_batch_allgather: call rf_comm_init first");
    const size_t img_bytes = (size_t)h->cfg.net_h * h->cfg.net_w * 3;
    try {
        CK(cudaSetDevice(h->device));
        ensure_slots(h);
        Ctx &c = h->ctx[h->submit_seq % h->ctx.size()];
        rf_handle_s::Slot &sl = h->slots[h->submit_seq % RF_PIPELINE_DEPTH];
        if (sl.busy) return fail(h, RF_ERR_CAPACITY, "rf_submit_batch: RF_PIPELINE_DEPTH batches already in flight; collect one first");
        H2DRuns runs{sl.d_in, img_bytes, h->copy_stream};     // H2D on the copy stream
        for (int i = 0; i < n; i++) {
            if (!imgs[i]) return fail(h, RF_ERR_INVALID_ARG, fmt("rf_submit_batch: image %d is NULL", i));
            const uint8_t *src = imgs[i];
            if (!is_pinned(src)) {
                memcpy(sl.h_in + (size_t)i * img_bytes, src, img_bytes);   // slot is free: its previous H2D completed before collect
                src = sl.h_in + (size_t)i * img_bytes;
            }
            runs.add(i, src);
        }
        runs.flush();
        CK(cudaEventRecord(sl.ev_h2d, h->copy_stream));
        CK(cudaStreamWaitEvent(c.stream, sl.ev_h2d, 0));
        if (c.param_seq && c.param_seq % Ctx::kParamSlots == 0) CK(cudaStreamSynchronize(c.stream));
        const unsigned seq = gather ? ++h->comm.seq : 0u;
        set_params(h, c, thr, nms, sl.d_in, seq);
        forward_graph(h, c, n);
        if (gather) {
            // results of ALL ranks: wait for every rank's flags of this step, then read this rank's window slot
            Comm::Slot &cs = h->comm.slots[h->submit_seq % RF_PIPELINE_DEPTH];
            const size_t nimg = (size_t)h->comm.world * h->cfg.max_batch;
            if (!cs.h_dets) {
                CK(cudaHostAlloc(&cs.h_dets, sizeof(rf_det) * nimg * h->cfg.max_faces, cudaHostAllocDefault));
                CK(cudaHostAlloc(&cs.h_counts, sizeof(int) * nimg, cudaHostAllocDefault));
            }
            const unsigned slot = seq % (unsigned)h->comm.ring;
            const size_t img0 = (size_t)slot * nimg;
            CK(cudaMemcpyAsync(cs.h_counts, c.pb.comm.counts[h->comm.rank] + img0, sizeof(int) * nimg, cudaMemcpyDeviceToHost, c.stream));
            CK(cudaMemcpyAsync(cs.h_dets, c.pb.comm.dets[h->comm.rank] + img0 * h->cfg.max_faces, sizeof(rf_det) * nimg * h->cfg.max_faces, cudaMemcpyDeviceToHost,
                               c.stream));
            CK(cudaMemcpyAsync(h->comm.h_err, h->comm.d_err, 4, cudaMemcpyDeviceToHost, c.stream));
        } else {
            CK(cudaMemcpyAsync(sl.h_counts, c.pb.out_counts, sizeof(int) * n, cudaMemcpyDeviceToHost, c.stream));
            CK(cudaMemcpyAsync(sl.h_dets, c.pb.out_dets, sizeof(rf_det) * (size_t)n * h->cfg.max_faces, cudaMemcpyDeviceToHost, c.stream));
        }
        CK(cudaEventRecord(sl.ev_done, c.stream));
        sl.n = n;
        sl.busy = true;
        sl.gather = gather;
        *ticket = (int)h->submit_seq++;
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_submit_batch(rf_handle h, const uint8_t *const *imgs, int n, float thr, float nms, int *ticket) {
    return submit_impl(h, imgs, n, thr, nms, ticket, false);
}
int rf_submit_batch_allgather(rf_handle h, const uint8_t *const *imgs, int n, float thr, float nms, int *ticket) {
    return submit_impl(h, imgs, n, thr, nms, ticket, true);
}

static int collect_impl(rf_handle h, int ticket, rf_face *out_faces, int *out_counts, int32_t *out_idx, bool gather) {
    if (!h) return RF_ERR_INVALID_ARG;
    if ((unsigned)ticket != h->collect_seq) return fail(h, RF_ERR_INVALID_ARG, fmt("rf_collect_batch: ticket %d out of order (next is %u)", ticket, h->collect_seq));
    rf_handle_s::Slot &sl = h->slots[h->collect_seq % RF_PIPELINE_DEPTH];
    if (!sl.busy) return fail(h, RF_ERR_INVALID_ARG, "rf_collect_batch: nothing submitted under this ticket");
    if (sl.gather != gather) return fail(h, RF_ERR_INVALID_ARG, "rf_collect_batch: ticket was submitted with the other (all-gather / local) entry point");
    try {
        CK(cudaSetDevice(h->device));
        CK(cudaEventSynchronize(sl.ev_done));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    sl.busy = false;
    h->collect_seq++;
    if (!gather) {
        put_results(h, sl.h_dets, sl.h_counts, 0, sl.n, out_faces, out_counts, out_idx);
        return RF_OK;
    }
    const Comm::Slot &cs = h->comm.slots[(unsigned)ticket % RF_PIPELINE_DEPTH];
    if (*h->comm.h_err) return fail(h, RF_ERR_CUDA, fmt("multi-GPU exchange: rank %u never delivered its records of this step", *h->comm.h_err - 1));
    // rank r's image i at r * max_batch + i; images beyond a rank's n are reported empty
    const size_t mb = h->cfg.max_batch;
    for (int r = 0; r < h->comm.world; r++) {
        put_results(h, cs.h_dets, cs.h_counts, r * mb, sl.n, out_faces, out_counts, out_idx);
        if (out_counts) std::fill(out_counts + r * mb + sl.n, out_counts + (r + 1) * mb, 0);
    }
    return RF_OK;
}

int rf_collect_batch(rf_handle h, int ticket, rf_face *out_faces, int *out_counts, int32_t *out_idx) {
    return collect_impl(h, ticket, out_faces, out_counts, out_idx, false);
}
int rf_collect_batch_allgather(rf_handle h, int ticket, rf_face *out_faces, int *out_counts, int32_t *out_idx) {
    return collect_impl(h, ticket, out_faces, out_counts, out_idx, true);
}
int rf_detect_batch_allgather(rf_handle h, const uint8_t *const *imgs, int n, float thr, float nms, rf_face *out_faces, int *out_counts, int32_t *out_idx) {
    int t = 0;
    int rc = rf_submit_batch_allgather(h, imgs, n, thr, nms, &t);
    if (rc) return rc;
    return rf_collect_batch_allgather(h, t, out_faces, out_counts, out_idx);
}

// rf_detect_views and rf_detect_views_oriented: view v is (shrink, LB_* bits); `views` only for the NULL check of either entry point
static int views_impl(rf_handle h, const char *who, const uint8_t *bgr, int width, int height, int row_stride, const void *views, int nviews,
                      const std::function<float(int)> &shrink_of, const std::function<int(int)> &bits_of, float thr, float nms, rf_face *out_faces,
                      int *out_count, int32_t *out_view_of, float *out_view_scales) {
    if (!h || !bgr || !views || !out_count || width <= 0 || height <= 0) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: bad arguments", who));
    if (nviews < 1 || nviews > RF_MAX_VIEWS || nviews > h->cfg.max_batch)
        return fail(h, RF_ERR_CAPACITY, fmt("%s: %d views, limit min(RF_MAX_VIEWS = %d, max_batch = %d)", who, nviews, RF_MAX_VIEWS, h->cfg.max_batch));
    const BgrImages src{&bgr, &width, &height, &row_stride, nullptr, false};
    int rc = src.check(h, who, 1);
    if (rc) return rc;
    for (int v = 0; v < nviews; v++) {
        const float shrink = shrink_of(v);
        if (!(shrink > 0.f && shrink <= 1.f)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: view %d: shrink must be in (0, 1]", who, v));
        if (bits_of(v) < 0) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: view %d: orientation must be in 1..8 (EXIF)", who, v));
    }
    static_assert(RF_MAX_VIEWS == RF_MAX_VIEWS_DEV, "view capacity of the merge kernel");
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w, mf = h->cfg.max_faces;
    const size_t img_bytes = (size_t)Hn * Wn * 3;
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        // every view may contribute max_faces candidates to the merged list of the one image
        if (!h->pb_merge.cand_keys) alloc_post_buffers(h->pb_merge, h->cfg.max_batch * mf, 1, mf);
        const BgrRows d_src = src.upload(h, c.stream, 0, 0);
        const int area = (h->cfg.flags & RF_FLAG_NPP_RESIZE) ? 1 : 0;
        std::vector<LbItem> lb(nviews);
        std::vector<MergeSource> ms(nviews);
        for (int v = 0; v < nviews; v++) {
            const int bw = std::max(1, (int)(Wn * shrink_of(v))), bh = std::max(1, (int)(Hn * shrink_of(v)));
            const int bits = bits_of(v);
            // the view letter-boxes the displayed image; its faces map back into stored pixels (postproc.cuh)
            const int dw = (bits & LB_TRANSPOSE) ? height : width, dh = (bits & LB_TRANSPOSE) ? width : height;
            const float scale = letterbox_fill(lb[v], d_src, dw, dh, h->d_input + (size_t)v * img_bytes, bw, bh, bits, area);
            ms[v] = (bits & ~LB_FLIP_X) ? oriented_view_source(v, mf, scale, bits, dw, dh) : view_source(v, mf, scale, bits, width);
            if (out_view_scales) out_view_scales[v] = scale;
        }
        CK(launch_letterbox_batch(lb.data(), nviews, Wn, Hn, c.stream));     // all views of the image: one launch
        set_params(h, c, thr, nms);
        forward_graph(h, c, nviews);
        CK(launch_merge(c.pb, ms.data(), nviews, Wn, Hn, h->pb_merge, c.stream));
        CK(launch_nms(1, c.d_params, h->pb_merge, c.stream));
        CK(cudaMemcpyAsync(h->h_counts, h->pb_merge.out_counts, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
        CK(cudaMemcpyAsync(h->h_dets, h->pb_merge.out_dets, sizeof(rf_det) * (size_t)mf, cudaMemcpyDeviceToHost, c.stream));
        CK(cudaStreamSynchronize(c.stream));
        const int k = h->h_counts[0];
        *out_count = k;
        for (int j = 0; j < k; j++) {
            if (out_faces) out_faces[j] = h->h_dets[j].face;
            if (out_view_of) out_view_of[j] = h->h_dets[j].anchor_index / mf;
        }
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_detect_views(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_view *views, int nviews, float thr,
                    float nms, rf_face *out_faces, int *out_count, int32_t *out_view_of, float *out_view_scales) {
    return views_impl(h, "rf_detect_views", bgr, width, height, row_stride, views, nviews, [&](int v) { return views[v].shrink; },
                      [&](int v) { return views[v].flip ? 1 : 0; }, thr, nms, out_faces, out_count, out_view_of, out_view_scales);
}

int rf_detect_views_oriented(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_oriented_view *views, int nviews,
                             float thr, float nms, rf_face *out_faces, int *out_count, int32_t *out_view_of, float *out_view_scales) {
    return views_impl(h, "rf_detect_views_oriented", bgr, width, height, row_stride, views, nviews, [&](int v) { return views[v].shrink; },
                      [&](int v) { return lb_orientation_bits(views[v].orientation); }, thr, nms, out_faces, out_count, out_view_of,
                      out_view_scales);
}

// ---- f23 rotated views (rf_b200.h rf_rotated_view) -------------------------------------------------------------------------------
static int check_rotated(rf_handle h, const char *who, float angle, float shrink, int v) {
    if (!std::isfinite(angle)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: view %d: the angle must be finite", who, v));
    if (!(shrink > 0.f && shrink <= 1.f)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: view %d: shrink must be in (0, 1]", who, v));
    return RF_OK;
}

// The shrink box of a view, as views_impl computes it
static void shrink_box(rf_handle h, float shrink, int &bw, int &bh) {
    bw = std::max(1, (int)(h->cfg.net_w * shrink));
    bh = std::max(1, (int)(h->cfg.net_h * shrink));
}

// The geometry of view (angle, shrink) of a width x height image
static RotatedGeometry view_geometry(rf_handle h, const rf_rotated_view &view, int width, int height) {
    int bw, bh;
    shrink_box(h, view.shrink, bw, bh);
    return rotated_geometry(view.angle, width, height, bw, bh);
}

// M of a view as the calls report it: all zero for a quarter turn
static void put_view_mat(const RotatedGeometry &g, double *out) {
    for (int k = 0; k < 6; k++) out[k] = g.orientation ? 0.0 : g.M[k];
}

extern "C++" {
// View v of image `image` into batch slot b, whose input is dst: a quarter turn appends rf_detect_views_oriented's letter-box item and
// merge source (its slot is b = w.lb.size()), a warp view a warp item and its rotated merge source.  width x height is the image's
// DISPLAYED size and `orient` its own LB_* bits (0: upright, the stored image; f25: the displayed frame D = T_o(S) of an oriented video):
// a quarter turn of D reads S through the composed orientation, a warp view reads D through f9's map, and either maps its faces back
// into D's pixels.  Returns the view's map-back scale: the letter-box's factor, or (float)(1 / f).
template <typename Src>
static float rotated_item(rf_handle h, const RotatedGeometry &g, float shrink, int v, int image, Src src, int width, int height, int orient,
                          int b, uint8_t *dst, ChunkWork<Src> &w) {
    const int mf = h->cfg.max_faces;
    if (g.orientation) {
        int bw, bh;
        shrink_box(h, shrink, bw, bh);
        const int bits = lb_orientation_bits(g.orientation);
        const int dw = (bits & LB_TRANSPOSE) ? height : width, dh = (bits & LB_TRANSPOSE) ? width : height;
        const int read = orient ? lb_orientation_bits(exif_compose(lb_exif(orient), g.orientation)) : bits;
        w.lb.emplace_back();
        const float scale = letterbox_fill(w.lb.back(), src, dw, dh, dst, bw, bh, read, (h->cfg.flags & RF_FLAG_NPP_RESIZE) ? 1 : 0);
        MergeSource m = (bits & ~LB_FLIP_X) ? oriented_view_source(v, mf, scale, bits, dw, dh) : view_source(v, mf, scale, bits, width);
        m.image = image;
        w.ms.push_back(m);
        return scale;
    }
    WarpItemT<Src> it{src, width, height, dst, {}};
    std::copy(g.iM, g.iM + 6, it.im);
    w.wp.push_back(it);
    w.wp_bits.push_back(orient);
    RotatedSource r{b, v * mf, image, {}, 1.0 / (2.0 * g.f)};
    std::copy(g.iM, g.iM + 6, r.im);
    w.rs.push_back(r);
    return (float)(1.0 / g.f);
}
}  // extern "C++"

int rf_detect_views_rotated(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_rotated_view *views, int nviews,
                            float thr, float nms, const rf_align_params *align, rf_face *out_faces, int *out_count, int32_t *out_view_of,
                            float *out_view_scales, double *out_view_mats, void *out_crops, double *out_mats) {
    const char *who = "rf_detect_views_rotated";
    if (!h || !bgr || !views || !out_count || width <= 0 || height <= 0) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: bad arguments", who));
    if (nviews < 1 || nviews > RF_MAX_VIEWS)
        return fail(h, RF_ERR_CAPACITY, fmt("%s: %d views, limit RF_MAX_VIEWS = %d", who, nviews, RF_MAX_VIEWS));
    const BgrImages src{&bgr, &width, &height, &row_stride, nullptr, false};
    int rc = src.check(h, who, 1);
    if (rc) return rc;
    for (int v = 0; v < nviews; v++)
        if ((rc = check_rotated(h, who, views[v].angle, views[v].shrink, v))) return rc;
    AlignArgs a;
    if (align && (rc = check_align(h, who, align, 1, out_crops, 1, a))) return rc;
    static_assert(RF_MAX_VIEWS == RF_MAX_VIEWS_DEV && RF_MAX_VIEWS == WARP_MAX_VIEWS, "view capacity of the warp and merge kernels");
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w, mf = h->cfg.max_faces, B = h->cfg.max_batch;
    const size_t img_bytes = (size_t)Hn * Wn * 3;
    // the quarter turns first: within a batch they take slots 0 .. k-1, as launch_merge reads them; ids keep the caller's order
    std::vector<RotatedGeometry> geo(nviews);
    std::vector<int> order;
    for (int v = 0; v < nviews; v++) {
        geo[v] = view_geometry(h, views[v], width, height);
        if (geo[v].orientation) order.push_back(v);
    }
    for (int v = 0; v < nviews; v++)
        if (!geo[v].orientation) order.push_back(v);
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        // every view may contribute max_faces candidates to the merged list of the one image
        if (h->pb_merge.anchors_per_image < RF_MAX_VIEWS * mf) {
            free_post_buffers(h->pb_merge);
            alloc_post_buffers(h->pb_merge, RF_MAX_VIEWS * mf, 1, mf);
        }
        const BgrRows d_src = src.upload(h, c.stream, 0, 0);
        set_params(h, c, thr, nms);
        for (int v0 = 0; v0 < nviews; v0 += B) {
            const int m = std::min(B, nviews - v0);
            ChunkWork<BgrRows> w;
            for (int b = 0; b < m; b++) {
                const int v = order[v0 + b];
                const float scale = rotated_item(h, geo[v], views[v].shrink, v, 0, d_src, width, height, 0, b, h->d_input + (size_t)b * img_bytes, w);
                if (out_view_scales) out_view_scales[v] = scale;
                if (out_view_mats) put_view_mat(geo[v], out_view_mats + (size_t)v * 6);
            }
            CK(launch_letterbox_batch(w.lb.data(), (int)w.lb.size(), Wn, Hn, c.stream));
            CK(launch_letterbox_warp(w.wp.data(), (int)w.wp.size(), Wn, Hn, c.stream));
            forward_graph(h, c, m);
            CK(launch_merge(c.pb, w.ms.data(), (int)w.ms.size(), Wn, Hn, h->pb_merge, c.stream));
            CK(launch_merge_rotated(c.pb, w.rs.data(), (int)w.rs.size(), h->pb_merge, c.stream));
        }
        CK(launch_nms(1, c.d_params, h->pb_merge, c.stream));
        if (align) {
            ensure_align_buffers(h, 1, a);
            a.n = 1;
            a.crops = h->d_align_crops;
            a.mats = out_mats ? h->d_align_mats : nullptr;
            const AlignImageT<BgrRows> orig{d_src, width, height, 1.f, 0};     // the merged records are in image pixels
            CK(launch_align_faces(a, &orig, h->pb_merge, h->num_sms, c.stream));
        }
        CK(cudaMemcpyAsync(h->h_counts, h->pb_merge.out_counts, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
        CK(cudaMemcpyAsync(h->h_dets, h->pb_merge.out_dets, sizeof(rf_det) * (size_t)mf, cudaMemcpyDeviceToHost, c.stream));
        CK(cudaStreamSynchronize(c.stream));
        const int k = h->h_counts[0];
        *out_count = k;
        for (int j = 0; j < k; j++) {
            if (out_faces) out_faces[j] = h->h_dets[j].face;
            if (out_view_of) out_view_of[j] = h->h_dets[j].anchor_index / mf;
        }
        const size_t nc = (size_t)std::min(k, align ? a.max_align : 0);
        if (nc) {
            CK(cudaMemcpy(out_crops, h->d_align_crops, nc * a.crop_bytes, cudaMemcpyDeviceToHost));
            if (out_mats) CK(cudaMemcpy(out_mats, h->d_align_mats, nc * 6 * sizeof(double), cudaMemcpyDeviceToHost));
        }
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

extern "C++" {
// The network input of one view of image 0 of src, either kind, into `out`, and its M (f23 / f24's parity hooks).
template <typename Source>
static int preprocess_rotated(rf_handle h, const char *who, const Source &src, float angle, float shrink, uint8_t *out, double *out_mat) {
    if (!h) return RF_ERR_INVALID_ARG;
    if (!out) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out is NULL", who));
    int rc = src.check(h, who, 1);
    if (rc || (rc = check_rotated(h, who, angle, shrink, 0))) return rc;
    const int Hn = h->cfg.net_h, Wn = h->cfg.net_w;
    const RotatedGeometry g = view_geometry(h, rf_rotated_view{angle, shrink}, src.width(0), src.height(0));
    try {
        CK(cudaSetDevice(h->device));
        cudaStream_t s = h->ctx[0].stream;
        ChunkWork<typename Source::Src> w;
        rotated_item(h, g, shrink, 0, 0, src.upload(h, s, 0, 0), src.width(0), src.height(0), 0, 0, h->d_input, w);
        CK(launch_letterbox_batch(w.lb.data(), (int)w.lb.size(), Wn, Hn, s));
        CK(launch_letterbox_warp(w.wp.data(), (int)w.wp.size(), Wn, Hn, s));
        CK(cudaMemcpyAsync(h->h_input, h->d_input, (size_t)Hn * Wn * 3, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        memcpy(out, h->h_input, (size_t)Hn * Wn * 3);
        if (out_mat) put_view_mat(g, out_mat);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}
}  // extern "C++"

int rf_preprocess_rotated(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, float angle, float shrink, uint8_t *out,
                          double *out_mat) {
    return preprocess_rotated(h, "rf_preprocess_rotated", BgrImages{&bgr, &width, &height, &row_stride, nullptr, false}, angle, shrink, out,
                              out_mat);
}

// ---- f24 rotated views of device frames (rf_b200.h) -----------------------------------------------------------------------------
extern "C++" {
// The jobs of a rotated device call: every view of each frame, geometry geo[i * nviews + v] of frame i's displayed size (f25: an
// oriented frame's views rotate D = T_o(S)).  Within a chunk the
// quarter turns take the first slots (launch_merge reads contiguous slots from 0); ids carry the caller's view index, so the slot
// order does not change a result.  Each job's map-back scale goes to scales[i * nviews + v].
template <typename Source>
struct RotatedJobs {
    rf_handle h;
    const Source &source;
    const rf_rotated_view *views;
    int nviews;
    const std::vector<RotatedGeometry> &geo;
    float *scales;
    int count(int) const { return nviews; }
    void fill(const Job *jobs, int m, const std::vector<typename Source::Src> &src, uint8_t *input, ChunkWork<typename Source::Src> &w) const {
        const size_t img_bytes = (size_t)h->cfg.net_h * h->cfg.net_w * 3;
        int b = 0;
        for (int warp = 0; warp < 2; warp++)
            for (int j = 0; j < m; j++) {
                const Job r = jobs[j];
                const size_t k = (size_t)r.image * nviews + r.item;
                if ((geo[k].orientation == 0) != (warp == 1)) continue;
                int dw, dh;
                displayed_size(source, r.image, dw, dh);
                scales[k] = rotated_item(h, geo[k], views[r.item].shrink, r.item, r.image, src[r.image], dw, dh, source.bits(r.image), b,
                                         input + (size_t)b * img_bytes, w);
                b++;
            }
    }
};

// The issue of a checked rotated device call of n > 0 frames into the rotated ring: each view's geometry of each frame's displayed
// size into geo, the map-back scales into scales.
template <typename Source>
static void rotated_issue(rf_handle h, const Source &source, int n, const rf_rotated_view *views, int nviews, float thr, float nms,
                          const AlignArgs *align, const rf_det **dev_dets, const int32_t **dev_counts, cudaEvent_t *free,
                          std::vector<RotatedGeometry> &geo, std::vector<float> &scales) {
    geo.resize((size_t)n * nviews);
    for (int i = 0; i < n; i++) {
        int dw, dh;
        displayed_size(source, i, dw, dh);
        for (int v = 0; v < nviews; v++) geo[(size_t)i * nviews + v] = view_geometry(h, views[v], dw, dh);
    }
    scales.resize(geo.size());
    device_issue(h, h->rotated_slots, h->next_rotated_slot, source, n, RotatedJobs<Source>{h, source, views, nviews, geo, scales.data()}, thr,
                 nms, align, dev_dets, dev_counts, free);
}

// rf_detect_views_rotated_device / rf_detect_yuv_views_rotated_device: the checks (the source, the views, then align), then the issue
// into the rotated ring.
template <typename Source>
static int detect_rotated_device(rf_handle h, const char *who, const Source &source, int n, const rf_rotated_view *views, int nviews, float thr,
                                 float nms, const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                                 const int32_t **dev_counts, float *out_view_scales, double *out_view_mats) {
    int rc = source.check(h, who, n);
    if (rc || (rc = rf_eng::rotated_views_check(h, who, views, nviews))) return rc;
    AlignArgs a;
    if (align && (rc = check_align(h, who, align, n, dev_crops, 0, a))) return rc;
    if (n == 0) return RF_OK;
    std::vector<RotatedGeometry> geo;
    std::vector<float> scales;
    a.crops = dev_crops;
    a.mats = dev_mats;
    try {
        rotated_issue(h, source, n, views, nviews, thr, nms, align ? &a : nullptr, dev_dets, dev_counts, nullptr, geo, scales);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    if (out_view_scales) std::copy(scales.begin(), scales.end(), out_view_scales);
    if (out_view_mats)
        for (size_t k = 0; k < geo.size(); k++) put_view_mat(geo[k], out_view_mats + k * 6);
    return RF_OK;
}

// The views of a rotated device call or a views tracker (f25), with f23 / f24's statuses and messages.
int rf_eng::rotated_views_check(rf_handle h, const char *who, const rf_rotated_view *views, int nviews) {
    if (!views) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: views is NULL", who));
    if (nviews < 1 || nviews > RF_MAX_VIEWS)
        return fail(h, RF_ERR_CAPACITY, fmt("%s: %d views, limit RF_MAX_VIEWS = %d", who, nviews, RF_MAX_VIEWS));
    for (int v = 0; v < nviews; v++) {
        const int rc = check_rotated(h, who, views[v].angle, views[v].shrink, v);
        if (rc) return rc;
    }
    return RF_OK;
}

// rf_detect_yuv_views_rotated_device's check and issue without crops, for the tracker's detect calls (tracker.cu, f25).
int rf_eng::yuv_rotated_check(rf_handle h, const char *who, const YuvFrames &src, int n, const rf_rotated_view *views, int nviews) {
    const int rc = src.check(h, who, n);
    return rc ? rc : rotated_views_check(h, who, views, nviews);
}

int rf_eng::yuv_rotated_issue(rf_handle h, const YuvFrames &src, int n, const rf_rotated_view *views, int nviews, float thr, float nms,
                              const rf_det **dev_dets, const int32_t **dev_counts, cudaEvent_t *free) {
    std::vector<RotatedGeometry> geo;
    std::vector<float> scales;
    try {
        rotated_issue(h, src, n, views, nviews, thr, nms, nullptr, dev_dets, dev_counts, free, geo, scales);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

}  // extern "C++"

int rf_detect_views_rotated_device(rf_handle h, const uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides,
                                   int n, const rf_rotated_view *views, int nviews, float thr, float nms, const rf_align_params *align,
                                   void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts, float *out_view_scales,
                                   double *out_view_mats) {
    return detect_rotated_device(h, "rf_detect_views_rotated_device", BgrImages{dev_bgr, widths, heights, row_strides, nullptr, false}, n,
                                 views, nviews, thr, nms, align, dev_crops, dev_mats, dev_dets, dev_counts, out_view_scales, out_view_mats);
}

int rf_detect_yuv_views_rotated_device(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_rotated_view *views, int nviews,
                                       float thr, float nms, const rf_align_params *align, void *dev_crops, double *dev_mats,
                                       const rf_det **dev_dets, const int32_t **dev_counts, float *out_view_scales, double *out_view_mats) {
    return detect_rotated_device(h, "rf_detect_yuv_views_rotated_device", YuvFrames{frames, matrix, nullptr, false}, n, views, nviews, thr,
                                 nms, align, dev_crops, dev_mats, dev_dets, dev_counts, out_view_scales, out_view_mats);
}

int rf_preprocess_yuv_rotated(rf_handle h, const rf_yuv_frame *frame, int matrix, float angle, float shrink, uint8_t *out, double *out_mat) {
    return preprocess_rotated(h, "rf_preprocess_yuv_rotated", YuvFrames{frame, matrix, nullptr, false}, angle, shrink, out, out_mat);
}

int rf_fetch_dets(rf_handle h, const rf_det *dev_dets, const int32_t *dev_counts, int n, rf_face *out_faces, int *out_counts,
                  int32_t *out_anchor_index) {
    int rc = check_n(h, n);
    if (rc || n == 0) return rc;
    if (!dev_dets || !dev_counts || !out_faces || !out_counts) return fail(h, RF_ERR_INVALID_ARG, "rf_fetch_dets: NULL records or outputs");
    try {
        CK(cudaSetDevice(h->device));
        for (Ctx &c : h->ctx) CK(cudaStreamSynchronize(c.stream));
        PostBuffers pb{};
        pb.out_dets = const_cast<rf_det *>(dev_dets);
        pb.out_counts = const_cast<int32_t *>(dev_counts);
        fetch_post(h, pb, h->ctx[0].stream, n, out_faces, out_counts, out_anchor_index);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

static void ensure_blobs(rf_handle h) {
    if (h->d_blobs[0]) return;
    for (int i = 0; i < 9; i++) CK(cudaMalloc(&h->d_blobs[i], sizeof(float) * h->blob_elems[i] * h->cfg.max_batch));
}

int rf_forward_heads(rf_handle h, const uint8_t *bgr, int n, float *const heads_out[9]) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (n == 0) return RF_OK;
    if (!bgr || !heads_out) return fail(h, RF_ERR_INVALID_ARG, "rf_forward_heads: NULL argument");
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        ensure_blobs(h);
        const size_t bytes = (size_t)n * h->cfg.net_h * h->cfg.net_w * 3;
        CK(cudaStreamSynchronize(c.stream));
        memcpy(h->h_input, bgr, bytes);
        CK(cudaMemcpyAsync(h->d_input, h->h_input, bytes, cudaMemcpyHostToDevice, c.stream));
        set_params(h, c, c.cur_thr, c.cur_nms);
        run_steps(h, Run{c, n, c.stream, h->d_blobs});
        CK(cudaGetLastError());
        for (int i = 0; i < 9; i++)
            CK(cudaMemcpyAsync(heads_out[i], h->d_blobs[i], sizeof(float) * h->blob_elems[i] * n, cudaMemcpyDeviceToHost, c.stream));
        CK(cudaStreamSynchronize(c.stream));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_postprocess(rf_handle h, const float *const heads[9], int n, float thr, float nms, rf_face *out_faces, int *out_counts,
                   int32_t *out_idx, int *out_ncand) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (n == 0) return RF_OK;
    if (!heads) return fail(h, RF_ERR_INVALID_ARG, "rf_postprocess: NULL heads");
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        ensure_blobs(h);
        for (int i = 0; i < 9; i++)
            CK(cudaMemcpyAsync(h->d_blobs[i], heads[i], sizeof(float) * h->blob_elems[i] * n, cudaMemcpyHostToDevice, c.stream));
        set_params(h, c, thr, nms);
        CK(launch_blob_decode(h->d_blobs, h->lv, n, h->cfg.net_w, h->cfg.net_h, c.d_params, c.pb, c.stream));
        if (out_ncand) CK(cudaMemcpyAsync(h->h_counts + h->cfg.max_batch, c.pb.cand_count, sizeof(int) * n, cudaMemcpyDeviceToHost, c.stream));
        CK(launch_nms(n, c.d_params, c.pb, c.stream));
        CK(cudaGetLastError());
        fetch_results(h, c, n, out_faces, out_counts, out_idx);
        if (out_ncand) for (int i = 0; i < n; i++) out_ncand[i] = h->h_counts[h->cfg.max_batch + i];
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// Debug / parity: any materialised activation by its Caffe top name, as NCHW float32.
int rf_debug_get_tensor(rf_handle h, const char *name, int n, float *out_nchw, int *c, int *hh, int *ww) {
    int rc = check_n(h, n);
    if (rc) return rc;
    auto it = h->tensor_by_name.find(name ? name : "");
    if (it == h->tensor_by_name.end()) return fail(h, RF_ERR_INVALID_ARG, fmt("unknown tensor '%s'", name ? name : "(null)"));
    const TensorInfo &t = h->tensors[it->second];
    if (c) *c = t.c;
    if (hh) *hh = t.h;
    if (ww) *ww = t.w;
    if (!out_nchw) return RF_OK;
    try {
        CK(cudaSetDevice(h->device));
        const Ctx &x = h->ctx[0];
        CK(cudaStreamSynchronize(x.stream));
        size_t elems = (size_t)n * t.h * t.w * t.c;
        std::vector<unsigned char> host(elems * h->elem);
        CK(cudaMemcpy(host.data(), x.arena + t.offset, host.size(), cudaMemcpyDeviceToHost));
        for (int b = 0; b < n; b++)
            for (int y = 0; y < t.h; y++)
                for (int x = 0; x < t.w; x++)
                    for (int ch = 0; ch < t.c; ch++) {
                        size_t src = (((size_t)b * t.h + y) * t.w + x) * t.c + ch;
                        float v = h->elem == 4 ? reinterpret_cast<float *>(host.data())[src]
                                : h->elem == 2 ? __half2float(reinterpret_cast<__half *>(host.data())[src])
                                               : (float)reinterpret_cast<int8_t *>(host.data())[src];   // INT8: raw quantised values
                        out_nchw[(((size_t)b * t.c + ch) * t.h + y) * t.w + x] = v;
                    }
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// Re-places activations without buffer reuse so that rf_debug_get_tensor sees every tensor of
// the last forward (debug only; call before the first forward).
int rf_debug_keep_all(rf_handle h) {
    if (!h) return RF_ERR_INVALID_ARG;
    try {
        CK(cudaSetDevice(h->device));
        for (auto &t : h->tensors) { t.first = -1; t.last = -1; }
        place_tensors(h, true);
        for (Ctx &c : h->ctx) {
            CK(cudaStreamSynchronize(c.stream));
            release_ctx(c, false);
            create_ctx(h, c, false);
        }
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// INT8 entropy calibration (SURVEY.md 8f-3; replaces INT8-Calibration-Tool/calibrationtable.cpp:399-583).  `h` must be an
// RF_PREC_FP32 handle (its SIMT plan materialises every tensor the INT8 plan quantises, including the depthwise outputs
// and the FPN sums).  Two passes over the n network-sized images: absmax, then 2048-bin histograms; then the KL threshold
// search per tensor on the host; the table is written in the reference's TensorRT cache format.
int rf_calibrate_int8(rf_handle h, const uint8_t *bgr_net_sized, int n_images, const char *out_table_path) {
    if (!h || !bgr_net_sized || n_images <= 0 || !out_table_path) return fail(h, RF_ERR_INVALID_ARG, "rf_calibrate_int8: bad arguments");
    if (h->cfg.precision != RF_PREC_FP32) return fail(h, RF_ERR_UNSUPPORTED, "rf_calibrate_int8: create the handle with RF_PREC_FP32 (every tensor must be materialised)");
    const size_t img_bytes = (size_t)h->cfg.net_h * h->cfg.net_w * 3;
    const int T = (int)h->tensors.size();
    float *d_max = nullptr;
    unsigned *d_hist = nullptr;
    try {
        CK(cudaSetDevice(h->device));
        int rc = rf_debug_keep_all(h);
        if (rc) return rc;
        Ctx &c = h->ctx[0];
        CK(cudaMalloc(&d_max, sizeof(float) * T));
        CK(cudaMalloc(&d_hist, sizeof(unsigned) * (size_t)T * CALIB_BINS));
        CK(cudaMemsetAsync(d_max, 0, sizeof(float) * T, c.stream));
        CK(cudaMemsetAsync(d_hist, 0, sizeof(unsigned) * (size_t)T * CALIB_BINS, c.stream));
        std::vector<float> hmax(T, 0.f);
        for (int pass = 0; pass < 2; pass++) {
            for (int i0 = 0; i0 < n_images; i0 += h->cfg.max_batch) {
                const int n = std::min(h->cfg.max_batch, n_images - i0);
                CK(cudaStreamSynchronize(c.stream));
                memcpy(h->h_input, bgr_net_sized + (size_t)i0 * img_bytes, (size_t)n * img_bytes);
                CK(cudaMemcpyAsync(h->d_input, h->h_input, (size_t)n * img_bytes, cudaMemcpyHostToDevice, c.stream));
                set_params(h, c, c.cur_thr, c.cur_nms);
                run_steps(h, Run{c, n, c.stream}, false);
                for (int t = 0; t < T; t++) {
                    const TensorInfo &ti = h->tensors[t];
                    const size_t elems = (size_t)n * ti.h * ti.w * ti.c;
                    const float *x = reinterpret_cast<const float *>(c.arena + ti.offset);
                    if (pass == 0) launch_absmax<float>(x, elems, d_max + t, c.stream);
                    else if (hmax[t] > 0.f) launch_hist<float>(x, elems, (float)CALIB_BINS / hmax[t], d_hist + (size_t)t * CALIB_BINS, c.stream);
                }
                CK(cudaGetLastError());
            }
            if (pass == 0) {
                CK(cudaMemcpyAsync(hmax.data(), d_max, sizeof(float) * T, cudaMemcpyDeviceToHost, c.stream));
                CK(cudaStreamSynchronize(c.stream));
            }
        }
        std::vector<unsigned> hist((size_t)T * CALIB_BINS);
        CK(cudaMemcpyAsync(hist.data(), d_hist, sizeof(unsigned) * hist.size(), cudaMemcpyDeviceToHost, c.stream));
        CK(cudaStreamSynchronize(c.stream));
        cudaFree(d_max); cudaFree(d_hist);
        d_max = nullptr; d_hist = nullptr;
        std::vector<std::pair<std::string, float>> scales;
        scales.emplace_back("data", 255.0f / 127.0f);          // u8 input range; the engine consumes the u8 image directly
        for (int t = 0; t < T; t++) {
            if (hmax[t] <= 0.f) { scales.emplace_back(h->tensors[t].name, 1.0f / 127.0f); continue; }
            const double bins = kl_threshold_bins(hist.data() + (size_t)t * CALIB_BINS);
            const double thr = bins * (double)hmax[t] / CALIB_BINS;
            scales.emplace_back(h->tensors[t].name, (float)(thr / 127.0));
        }
        std::string err;
        if (!write_int8_table(out_table_path, scales, err)) return fail(h, RF_ERR_IO, err);
    } catch (const CudaFail &f) {
        cudaFree(d_max); cudaFree(d_hist);
        return fail_cuda(h, f);
    }
    return RF_OK;
}

// Host-only: the KL threshold search on a caller-supplied histogram (for CPU-side tests of the calibrator).
double rf_kl_threshold_bins(const unsigned *hist, int bins, int levels) { return kl_threshold_bins(hist, bins, levels); }

// Host-only (no GPU needed): folded FP32 weights/bias of one convolution as the engine will hold
// them (BatchNorm + Scale + bias folded).  dims = {cout, cin/groups, k, k}.  Lets CPU-only tests
// check the model front end against the oracle's fold.
int rf_cache_status(rf_handle h) { return h ? h->cache_status : RF_ERR_INVALID_ARG; }

int rf_network_config(const char *network, int *num_levels, int strides[3], int scales[6], float ratios[2], int *num_ratios) {
    if (!network) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_network_config: NULL network");
    NetworkConfig nc;
    std::string err;
    const bool ok = network_config(network, nc, err);
    if (num_ratios) *num_ratios = (int)nc.ratios.size();
    if (ratios) for (size_t i = 0; i < nc.ratios.size() && i < 2; i++) ratios[i] = nc.ratios[i];
    if (!ok) return fail(nullptr, RF_ERR_UNSUPPORTED, err);
    if (num_levels) *num_levels = (int)nc.strides.size();
    for (size_t l = 0; l < nc.strides.size() && l < 3; l++) {
        if (strides) strides[l] = nc.strides[l];
        if (scales) { scales[2 * l] = nc.scales[l][0]; scales[2 * l + 1] = nc.scales[l][1]; }
    }
    return RF_OK;
}

int rf_model_load(const char *caffemodel_path, const char *prototxt_path, const char *cache_path, int *cache_status, int input_dims[4],
                  const char *layer, float *w, int wcap, float *b, int bcap, int dims[4]) {
    if (!caffemodel_path) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_model_load: NULL caffemodel_path");
    Model m;
    NetGraph g;
    std::string err;
    int st = RF_OK, cs = CACHE_NONE;
    if (!load_model(caffemodel_path, prototxt_path ? prototxt_path : "", cache_path ? cache_path : "", m, &g, &cs, err, st)) return fail(nullptr, st, err);
    if (cache_status) *cache_status = cs;
    if (input_dims) for (int k = 0; k < 4; k++) input_dims[k] = g.input_dims[k];
    if (!layer) return RF_OK;
    auto it = m.convs.find(layer);
    if (it == m.convs.end()) return fail(nullptr, RF_ERR_INVALID_ARG, std::string("no convolution '") + layer + "'");
    const FoldedConv &c = it->second;
    if (dims) { dims[0] = c.cout; dims[1] = c.cin / c.groups; dims[2] = c.k; dims[3] = c.k; }
    if (w) { if ((size_t)wcap < c.w.size()) return fail(nullptr, RF_ERR_CAPACITY, "w buffer too small"); memcpy(w, c.w.data(), c.w.size() * 4); }
    if (b) { if ((size_t)bcap < c.b.size()) return fail(nullptr, RF_ERR_CAPACITY, "b buffer too small"); memcpy(b, c.b.data(), c.b.size() * 4); }
    return RF_OK;
}

int rf_model_inspect(const char *caffemodel_path, const char *layer, float *w, int wcap, float *b, int bcap, int dims[4]) {
    if (!caffemodel_path || !layer) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_model_inspect: NULL argument");
    std::vector<RawLayer> layers;
    std::string err;
    bool io = false;
    Model m;
    if (!read_caffemodel(caffemodel_path, layers, err, io)) return fail(nullptr, io ? RF_ERR_IO : RF_ERR_MODEL, err);
    if (!build_mnet_model(layers, m, err)) return fail(nullptr, RF_ERR_MODEL, err);
    auto it = m.convs.find(layer);
    if (it == m.convs.end()) return fail(nullptr, RF_ERR_INVALID_ARG, std::string("no convolution '") + layer + "'");
    const FoldedConv &c = it->second;
    if (dims) { dims[0] = c.cout; dims[1] = c.cin / c.groups; dims[2] = c.k; dims[3] = c.k; }
    if (w) { if ((size_t)wcap < c.w.size()) return fail(nullptr, RF_ERR_CAPACITY, "w buffer too small"); memcpy(w, c.w.data(), c.w.size() * 4); }
    if (b) { if ((size_t)bcap < c.b.size()) return fail(nullptr, RF_ERR_CAPACITY, "b buffer too small"); memcpy(b, c.b.data(), c.b.size() * 4); }
    return RF_OK;
}

// Host-only (works without a GPU): builds the layer plan rf_create would build for `cfg` and writes one line per kernel
// launch of a forward, "step lane <lane>: <name>" and, where the launch is tiled, " | " and its tile geometry (and, for tile
// chains, their geometry and shared-memory budget) into `out`.
int rf_plan_describe(const rf_config *cfg, char *out, int cap) {
    if (!cfg || !cfg->caffemodel_path || !out || cap <= 0) return fail(nullptr, RF_ERR_INVALID_ARG, "rf_plan_describe: bad arguments");
    if (cfg->net_w <= 0 || cfg->net_h <= 0 || cfg->net_w % 32 || cfg->net_h % 32 || cfg->max_batch <= 0)
        return fail(nullptr, RF_ERR_INVALID_ARG, "rf_plan_describe: bad network size / batch");
    std::unique_ptr<rf_handle_s> H(new rf_handle_s);
    rf_handle h = H.get();
    h->cfg = *cfg;
    if (h->cfg.max_faces <= 0) h->cfg.max_faces = 256;
    h->elem = cfg->precision == RF_PREC_FP32 ? 4 : (cfg->precision == RF_PREC_FP16 ? 2 : 1);
    std::vector<RawLayer> layers;
    std::string err;
    bool io = false;
    if (!read_caffemodel(cfg->caffemodel_path, layers, err, io)) return fail(nullptr, io ? RF_ERR_IO : RF_ERR_MODEL, err);
    if (!build_mnet_model(layers, h->model, err)) return fail(nullptr, RF_ERR_MODEL, err);
    if (cfg->int8_table_path && !read_int8_table(cfg->int8_table_path, h->int8_scales, err)) return fail(nullptr, RF_ERR_IO, err);
    try {
        make_plan(h, false);
    } catch (const CudaFail &f) { return fail_cuda(nullptr, f); }
    catch (const PlanFail &f) { return fail(nullptr, f.status, f.msg); }
    std::string text = fmt("%d launches per forward, activation arena %zu bytes per batch of %d\n", (int)h->steps.size(), h->arena_bytes, cfg->max_batch);
    for (auto &st : h->steps) text += fmt("step lane %d: %s%s%s\n", st.lane, st.name.c_str(), st.geom.empty() ? "" : " | ", st.geom.c_str());
    text += describe_chains(h);
    snprintf(out, (size_t)cap, "%s", text.c_str());
    return (int)h->steps.size();
}

int rf_profile_layers(rf_handle h, int n, int iters, char (*names)[64], float *ms, double *bytes, double *flops, int cap) {
    int rc = check_n(h, n);
    if (rc) return rc;
    if (n == 0 || iters <= 0) return fail(h, RF_ERR_INVALID_ARG, "rf_profile_layers: n and iters must be positive");
    int cnt = 0;
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        set_params(h, c, c.cur_thr, c.cur_nms);
        run_steps(h, Run{c, n, c.stream}, false);  // warm everything once (also leaves consistent inputs for every step)
        CK(cudaStreamSynchronize(c.stream));
        const Run one{c, n, c.stream, nullptr, true};
        for (size_t si = 0; si < h->steps.size() && cnt < cap; si++) {
            const Step &st = h->steps[si];
            st.launch(one);
            CK(cudaEventRecord(h->ev0, c.stream));
            for (int i = 0; i < iters; i++) st.launch(one);
            CK(cudaEventRecord(h->ev1, c.stream));
            CK(cudaEventSynchronize(h->ev1));
            float t = 0;
            CK(cudaEventElapsedTime(&t, h->ev0, h->ev1));
            snprintf(names[cnt], 64, "%s", st.name.c_str());
            ms[cnt] = t / iters;
            if (bytes) bytes[cnt] = st.bytes_per_img * n;
            if (flops) flops[cnt] = st.flops_per_img * n;
            cnt++;
        }
        CK(cudaGetLastError());
        // single steps were launched out of their forward: leave the last-block / candidate counters as a forward expects them
        CK(cudaMemsetAsync(c.pb.tile_done, 0, sizeof(int) * h->cfg.max_batch, c.stream));
        CK(cudaMemsetAsync(c.pb.cand_count, 0, sizeof(int) * h->cfg.max_batch, c.stream));
        CK(cudaStreamSynchronize(c.stream));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return cnt;
}

}  // extern "C"

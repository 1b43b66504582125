// jpeg.cu -- f1 ingest, the half the reference does with cv::imread on the host (retinaface/main.cpp:18-26, :33-41): compressed
// JPEG bytes in, decoded BGR u8 pixels in DEVICE memory out, so that a camera-sized photo crosses PCIe as ~0.2 MB of
// bitstream instead of 3.4 MB of pixels (at batch 32 the end-to-end rate of the pixel path sits on the PCIe ceiling).
//
// The decoder is NVIDIA's nvJPEG -- a library call, like cv::imread is one in the reference; it is ingest, not the hot path.
// libnvjpeg.so.12 is opened at run time (dlopen), the way comm.cu opens NCCL: a deployment without it loses only
// rf_detect_jpeg_batch / rf_decode_jpeg, which then return RF_ERR_UNSUPPORTED.  Back ends, in order of preference (auto):
//   hardware        the NVJPG engines through nvjpegDecodeBatched (baseline, single scan) -- where nvJPEG offers them
//                   (nvjpegCreateEx(HARDWARE) fails where it does not)
//   default         nvjpegDecode (hybrid: Huffman on the host, IDCT + colour conversion + BGR interleave on the GPU), the images
//                   of a call spread over RF_JPEG_THREADS host threads (default: half the cores, at most 16)
// RF_JPEG_BACKEND = hardware | gpu_hybrid | hybrid_batched forces one of nvJPEG's batched decoders (measurements: all of them
// run at the single-thread Huffman rate at batch 8), = default skips them.
// Output format NVJPEG_OUTPUT_BGRI = the cv::Mat layout the rest of the path consumes (packed rows, pitch = 3 * width).
#include <dlfcn.h>
#include <nvjpeg.h>

#include <algorithm>
#include <cstring>
#include <thread>

#include "engine_internal.cuh"

namespace rf_eng {

namespace {

struct Api {
    void *lib = nullptr;
    nvjpegStatus_t (*CreateEx)(nvjpegBackend_t, nvjpegDevAllocator_t *, nvjpegPinnedAllocator_t *, unsigned int, nvjpegHandle_t *) = nullptr;
    nvjpegStatus_t (*Destroy)(nvjpegHandle_t) = nullptr;
    nvjpegStatus_t (*StateCreate)(nvjpegHandle_t, nvjpegJpegState_t *) = nullptr;
    nvjpegStatus_t (*StateDestroy)(nvjpegJpegState_t) = nullptr;
    nvjpegStatus_t (*GetImageInfo)(nvjpegHandle_t, const unsigned char *, size_t, int *, nvjpegChromaSubsampling_t *, int *, int *) = nullptr;
    nvjpegStatus_t (*Decode)(nvjpegHandle_t, nvjpegJpegState_t, const unsigned char *, size_t, nvjpegOutputFormat_t, nvjpegImage_t *, cudaStream_t) = nullptr;
    nvjpegStatus_t (*BatchedInitialize)(nvjpegHandle_t, nvjpegJpegState_t, int, int, nvjpegOutputFormat_t) = nullptr;
    nvjpegStatus_t (*Batched)(nvjpegHandle_t, nvjpegJpegState_t, const unsigned char *const *, const size_t *, nvjpegImage_t *, cudaStream_t) = nullptr;
};

struct Batched {                                       // one back end driven through nvjpegDecodeBatched
    const char *name;
    nvjpegBackend_t id;
    nvjpegHandle_t handle = nullptr;
    nvjpegJpegState_t state = nullptr;
    int batch = 0;                                     // batch size the state is initialised for
};
struct Codec {
    Api api;
    std::vector<Batched> batched;                      // in order of preference; only the ones this device / library offers
    nvjpegHandle_t def = nullptr;                      // default back end, image by image: takes whatever the batched ones refuse
    nvjpegJpegState_t def_state = nullptr;
    // nvJPEG's Huffman stage runs on the calling host thread (whatever the back end or the batch size), so the images of a call are spread over worker threads, each with its own decoder state and
    // stream (the library handle is thread safe, a state is not)
    struct Worker { nvjpegJpegState_t state = nullptr; cudaStream_t stream = nullptr; cudaEvent_t done = nullptr; };
    std::vector<Worker> workers;
    cudaEvent_t ready = nullptr;                       // the caller's stream has reached the point where the buffers are free
    int cpu_threads = 1;
    std::string backend = "none", last_used = "none";
};

const char *status_name(nvjpegStatus_t s) {
    switch (s) {
        case NVJPEG_STATUS_SUCCESS: return "success";
        case NVJPEG_STATUS_NOT_INITIALIZED: return "not initialised";
        case NVJPEG_STATUS_INVALID_PARAMETER: return "invalid parameter";
        case NVJPEG_STATUS_BAD_JPEG: return "bad JPEG";
        case NVJPEG_STATUS_JPEG_NOT_SUPPORTED: return "JPEG not supported";
        case NVJPEG_STATUS_ALLOCATOR_FAILURE: return "allocator failure";
        case NVJPEG_STATUS_EXECUTION_FAILED: return "execution failed";
        case NVJPEG_STATUS_ARCH_MISMATCH: return "architecture mismatch";
        case NVJPEG_STATUS_INTERNAL_ERROR: return "internal error";
        case NVJPEG_STATUS_IMPLEMENTATION_NOT_SUPPORTED: return "implementation not supported";
        default: return "incomplete bitstream / unknown";
    }
}

template <typename F>
bool sym(void *lib, const char *name, F &fn) {
    fn = reinterpret_cast<F>(dlsym(lib, name));
    return fn != nullptr;
}

// opens the library and creates the decoder handles once per rf handle; RF status
int codec(rf_handle h, Codec **out) {
    if (h->jpeg) { *out = static_cast<Codec *>(h->jpeg); return RF_OK; }
    Codec *c = new Codec();
    for (const char *name : {"libnvjpeg.so.12", "libnvjpeg.so"}) {
        c->api.lib = dlopen(name, RTLD_NOW | RTLD_LOCAL);
        if (c->api.lib) break;
    }
    if (!c->api.lib) { delete c; return fail(h, RF_ERR_UNSUPPORTED, "libnvjpeg.so.12 not found: JPEG ingest is unavailable (pixel entry points are unaffected)"); }
    Api &a = c->api;
    const bool ok = sym(a.lib, "nvjpegCreateEx", a.CreateEx) && sym(a.lib, "nvjpegDestroy", a.Destroy) && sym(a.lib, "nvjpegJpegStateCreate", a.StateCreate) &&
                    sym(a.lib, "nvjpegJpegStateDestroy", a.StateDestroy) && sym(a.lib, "nvjpegGetImageInfo", a.GetImageInfo) && sym(a.lib, "nvjpegDecode", a.Decode) &&
                    sym(a.lib, "nvjpegDecodeBatchedInitialize", a.BatchedInitialize) && sym(a.lib, "nvjpegDecodeBatched", a.Batched);
    if (!ok) { dlclose(a.lib); delete c; return fail(h, RF_ERR_UNSUPPORTED, "libnvjpeg lacks an entry point this library needs"); }
    // RF_JPEG_BACKEND: auto (default) | hardware | gpu_hybrid | hybrid_batched | default   -- anything but auto/default forces one
    const char *env = getenv("RF_JPEG_BACKEND");
    const std::string want = env ? env : "auto";
    nvjpegStatus_t s = a.CreateEx(NVJPEG_BACKEND_DEFAULT, nullptr, nullptr, 0, &c->def);
    if (s == NVJPEG_STATUS_SUCCESS) s = a.StateCreate(c->def, &c->def_state);
    if (s != NVJPEG_STATUS_SUCCESS) {
        const std::string msg = fmt("nvjpegCreateEx(default back end): %s", status_name(s));
        if (c->def) a.Destroy(c->def);
        dlclose(a.lib); delete c;
        return fail(h, RF_ERR_CUDA, msg);
    }
    {
        const char *te = getenv("RF_JPEG_THREADS");
        const int want_t = te ? atoi(te) : (int)(std::thread::hardware_concurrency() / 2);
        c->cpu_threads = std::max(1, std::min(16, want_t));
    }
    bool workers_ok = cudaEventCreateWithFlags(&c->ready, cudaEventDisableTiming) == cudaSuccess;
    for (int t = 0; workers_ok && t < c->cpu_threads; t++) {
        Codec::Worker wk;
        workers_ok = a.StateCreate(c->def, &wk.state) == NVJPEG_STATUS_SUCCESS && cudaStreamCreateWithFlags(&wk.stream, cudaStreamNonBlocking) == cudaSuccess &&
                     cudaEventCreateWithFlags(&wk.done, cudaEventDisableTiming) == cudaSuccess;
        c->workers.push_back(wk);
    }
    if (!workers_ok) {
        for (auto &wk : c->workers) { if (wk.state) a.StateDestroy(wk.state); if (wk.stream) cudaStreamDestroy(wk.stream); if (wk.done) cudaEventDestroy(wk.done); }
        a.StateDestroy(c->def_state); a.Destroy(c->def); dlclose(a.lib); delete c;
        return fail(h, RF_ERR_CUDA, "JPEG ingest: could not create the decoder worker states");
    }
    const Batched cands[] = {{"hardware", NVJPEG_BACKEND_HARDWARE}, {"gpu_hybrid", NVJPEG_BACKEND_GPU_HYBRID}, {"hybrid_batched", NVJPEG_BACKEND_HYBRID}};
    for (const Batched &cand : cands) {
        const bool forced = want == cand.name;
        // auto: the hardware engines when nvJPEG offers them; the other batched back ends only on request (they decode at
        // the single-thread Huffman rate whatever the batch size)
        if (!(forced || (want == "auto" && cand.id == NVJPEG_BACKEND_HARDWARE))) continue;
        Batched b = cand;
        if (a.CreateEx(b.id, nullptr, nullptr, 0, &b.handle) == NVJPEG_STATUS_SUCCESS && a.StateCreate(b.handle, &b.state) == NVJPEG_STATUS_SUCCESS) {
            c->batched.push_back(b);
        } else {
            if (b.handle) a.Destroy(b.handle);
            cudaGetLastError();
            if (forced) {
                a.StateDestroy(c->def_state); a.Destroy(c->def); dlclose(a.lib); delete c;
                return fail(h, RF_ERR_UNSUPPORTED, fmt("RF_JPEG_BACKEND=%s: nvJPEG cannot create that back end on this device", cand.name));
            }
        }
    }
    c->backend = c->batched.empty() ? "default" : c->batched[0].name;
    h->jpeg = c;
    *out = c;
    return RF_OK;
}

}  // namespace

void jpeg_release(rf_handle h) {
    if (!h->jpeg) return;
    Codec *c = static_cast<Codec *>(h->jpeg);
    for (Batched &b : c->batched) { c->api.StateDestroy(b.state); c->api.Destroy(b.handle); }
    for (auto &wk : c->workers) { cudaStreamSynchronize(wk.stream); c->api.StateDestroy(wk.state); cudaStreamDestroy(wk.stream); cudaEventDestroy(wk.done); }
    if (c->ready) cudaEventDestroy(c->ready);
    if (c->def_state) c->api.StateDestroy(c->def_state);
    if (c->def) c->api.Destroy(c->def);
    if (c->api.lib) dlclose(c->api.lib);
    delete c;
    h->jpeg = nullptr;
}

const char *jpeg_backend(rf_handle h) {
    static thread_local std::string s;
    if (!h->jpeg) return "none";
    Codec *c = static_cast<Codec *>(h->jpeg);
    s = c->backend + " (last call: " + c->last_used + ")";
    return s.c_str();
}

int jpeg_info(rf_handle h, const uint8_t *data, size_t len, int *w, int *hgt) {
    Codec *c = nullptr;
    int rc = codec(h, &c);
    if (rc) return rc;
    int ncomp = 0, ws[NVJPEG_MAX_COMPONENT] = {0}, hs[NVJPEG_MAX_COMPONENT] = {0};
    nvjpegChromaSubsampling_t ss;
    const nvjpegStatus_t s = c->api.GetImageInfo(c->def, data, len, &ncomp, &ss, ws, hs);
    if (s != NVJPEG_STATUS_SUCCESS) return fail(h, RF_ERR_INVALID_ARG, fmt("not a decodable JPEG stream (nvjpegGetImageInfo: %s)", status_name(s)));
    *w = ws[0]; *hgt = hs[0];
    return RF_OK;
}

// Decodes image i into dst[i] (device memory, packed BGR rows of w[i] pixels) on stream s.  The hardware engines take the
// whole batch in one call; streams they refuse (progressive, 4:1:0 ...) and devices without engines use the default back end
// image by image.
int jpeg_decode(rf_handle h, const uint8_t *const *data, const size_t *len, int n, uint8_t *const *dst, const int *w, const int *hgt, cudaStream_t s) {
    Codec *c = nullptr;
    int rc = codec(h, &c);
    if (rc) return rc;
    Api &a = c->api;
    std::vector<nvjpegImage_t> out(n);
    for (int i = 0; i < n; i++) {
        memset(&out[i], 0, sizeof(nvjpegImage_t));
        out[i].channel[0] = dst[i];
        out[i].pitch[0] = (size_t)w[i] * 3;
    }
    (void)hgt;
    for (Batched &b : c->batched) {
        nvjpegStatus_t st = NVJPEG_STATUS_SUCCESS;
        if (b.batch != n) {
            st = a.BatchedInitialize(b.handle, b.state, n, std::min(n, c->cpu_threads), NVJPEG_OUTPUT_BGRI);
            b.batch = st == NVJPEG_STATUS_SUCCESS ? n : 0;
        }
        if (st == NVJPEG_STATUS_SUCCESS) st = a.Batched(b.handle, b.state, data, len, out.data(), s);
        if (st == NVJPEG_STATUS_SUCCESS) { c->last_used = b.name; return RF_OK; }
        b.batch = 0;                     // a failed batch must be re-initialised; try the next back end
        cudaGetLastError();
    }
    const int T = std::min(n, (int)c->workers.size());
    if (T <= 1) {
        for (int i = 0; i < n; i++) {
            const nvjpegStatus_t st = a.Decode(c->def, c->def_state, data[i], len[i], NVJPEG_OUTPUT_BGRI, &out[i], s);
            if (st != NVJPEG_STATUS_SUCCESS) return fail(h, RF_ERR_INVALID_ARG, fmt("JPEG %d does not decode (nvjpegDecode: %s)", i, status_name(st)));
        }
        c->last_used = "default";
        return RF_OK;
    }
    // worker t decodes images t, t + T, ... on its own stream, behind the caller's stream (the destination buffers may still
    // be read by earlier work there); the caller's stream then waits for every worker
    if (cudaEventRecord(c->ready, s) != cudaSuccess) return fail(h, RF_ERR_CUDA, "JPEG ingest: cudaEventRecord failed");
    std::vector<nvjpegStatus_t> bad(T, NVJPEG_STATUS_SUCCESS);
    std::vector<int> bad_at(T, -1);
    std::vector<cudaError_t> cerr(T, cudaSuccess);
    std::vector<std::thread> th;
    const int device = h->device;
    for (int t = 0; t < T; t++)
        th.emplace_back([&, t]() {
            Codec::Worker &wk = c->workers[t];
            cerr[t] = cudaSetDevice(device);
            if (cerr[t] == cudaSuccess) cerr[t] = cudaStreamWaitEvent(wk.stream, c->ready, 0);
            for (int i = t; i < n && cerr[t] == cudaSuccess && bad[t] == NVJPEG_STATUS_SUCCESS; i += T) {
                const nvjpegStatus_t st = a.Decode(c->def, wk.state, data[i], len[i], NVJPEG_OUTPUT_BGRI, &out[i], wk.stream);
                if (st != NVJPEG_STATUS_SUCCESS) { bad[t] = st; bad_at[t] = i; }
            }
            if (cerr[t] == cudaSuccess) cerr[t] = cudaEventRecord(wk.done, wk.stream);
        });
    for (auto &x : th) x.join();
    for (int t = 0; t < T; t++) {
        if (cerr[t] == cudaSuccess) cerr[t] = cudaStreamWaitEvent(s, c->workers[t].done, 0);
        if (cerr[t] != cudaSuccess) return fail(h, RF_ERR_CUDA, fmt("JPEG ingest worker %d: %s", t, cudaGetErrorString(cerr[t])));
    }
    for (int t = 0; t < T; t++)
        if (bad[t] != NVJPEG_STATUS_SUCCESS) return fail(h, RF_ERR_INVALID_ARG, fmt("JPEG %d does not decode (nvjpegDecode: %s)", bad_at[t], status_name(bad[t])));
    c->last_used = fmt("default x %d threads", T);
    return RF_OK;
}

}  // namespace rf_eng

// f9: the Exif orientation cv::imread applies.  Walks the marker segments up to the first scan; in the first APP1 segment that
// starts "Exif\0\0" reads IFD0's tag 0x0112 (its first 16-bit value, as OpenCV's ExifReader does, whatever the declared type) in the
// TIFF header's byte order.  Every read is bounds-checked against the segment, and the segment against `bytes`.
extern "C" int rf_jpeg_exif_orientation(const uint8_t *p, size_t n) {
    if (!p || n < 4 || p[0] != 0xFF || p[1] != 0xD8) return 1;
    size_t i = 2;
    while (i + 4 <= n) {
        if (p[i] != 0xFF) return 1;
        const uint8_t m = p[i + 1];
        if (m == 0xFF) { i++; continue; }                                        // fill byte
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) { i += 2; continue; }          // markers without a length
        if (m == 0xDA || m == 0xD9) return 1;                                     // scan data / end of image: no Exif before it
        const size_t len = ((size_t)p[i + 2] << 8) | p[i + 3];
        if (len < 2 || i + 2 + len > n) return 1;
        if (m == 0xE1 && len >= 8 && memcmp(p + i + 4, "Exif\0\0", 6) == 0) {
            const uint8_t *t = p + i + 10;
            const size_t tn = len - 8;
            if (tn < 8) return 1;
            const bool le = t[0] == 'I' && t[1] == 'I', be = t[0] == 'M' && t[1] == 'M';
            if (!le && !be) return 1;
            auto u16 = [&](size_t o) -> unsigned { return le ? t[o] | (t[o + 1] << 8) : (t[o] << 8) | t[o + 1]; };
            auto u32 = [&](size_t o) -> size_t { return le ? (size_t)u16(o) | ((size_t)u16(o + 2) << 16) : ((size_t)u16(o) << 16) | u16(o + 2); };
            if (u16(2) != 42) return 1;
            const size_t ifd = u32(4);
            if (ifd > tn || tn - ifd < 2) return 1;
            const size_t cnt = u16(ifd);
            for (size_t k = 0; k < cnt; k++) {
                const size_t e = ifd + 2 + 12 * k;
                if (e > tn || tn - e < 12) return 1;
                if (u16(e) == 0x0112) {
                    const unsigned o = u16(e + 8);
                    return o >= 1 && o <= 8 ? (int)o : 1;
                }
            }
            return 1;
        }
        i += 2 + len;
    }
    return 1;
}

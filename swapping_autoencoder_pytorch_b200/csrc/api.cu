// C-ABI glue: globals, error reporting, conv entry points and kernel selection.
#include "conv_internal.cuh"
#include <mutex>

namespace sae {

thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};

int sm_count() {
    static int n = 0;
    static std::once_flag once;
    std::call_once(once, [] {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, dev) == cudaSuccess) n = prop.multiProcessorCount;
        if (n <= 0) n = 132;
    });
    return n;
}

static int validate_geom(const sae_conv_geom* g, const char* who) {
    if (!g) return fail(SAE_E_INVALID, "%s: null geometry", who);
    if (g->N < 0 || g->H <= 0 || g->W <= 0 || g->C <= 0 || g->K <= 0 || g->R <= 0 || g->S <= 0 || g->P <= 0 ||
        g->Q <= 0 || g->stride <= 0)
        return fail(SAE_E_INVALID, "%s: non-positive dimension", who);
    // the last output row/column must start inside the padded input
    if ((int64_t)(g->P - 1) * g->stride - g->pad_t + g->R - 1 < 0 || (int64_t)(g->Q - 1) * g->stride - g->pad_l + g->S - 1 < 0)
        return fail(SAE_E_INVALID, "%s: inconsistent P/Q", who);
    return SAE_OK;
}

}  // namespace sae

using namespace sae;

extern "C" int sae_abi_version(void) { return SAE_ABI_VERSION; }
extern "C" const char* sae_last_error(void) { return g_err; }
extern "C" int64_t sae_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
extern "C" int sae_tcgen05_available(void) { return tc_available() ? 1 : 0; }

extern "C" int sae_conv2d_query_impl(const sae_conv_geom* g, int dir) {
    if (validate_geom(g, "query_impl") != SAE_OK) return SAE_E_INVALID;
    if (!tc_available()) return 1;
    bool ok = dir == 0 ? tc_fprop_eligible(g) : dir == 1 ? tc_dgrad_eligible(g) : wgrad_wg_eligible(g);
    return ok ? 2 : 1;
}

// ws_bytes non-null: the deterministic twin (workspace protocol of det_workspace).  It takes the wgmma kernels wherever the
// shape qualifies without asking the device — the size query makes no CUDA call, and the library runs on sm_90a only — and
// only the generic kernel's split K has a reduction to make deterministic.
// w_lo non-null: the split-TF32 twin (filter pair (w, w_lo)); the TF32 entry points pass nullptr
static int conv2d_fprop(const float* x, const float* w, const float* w_lo, float* y, const sae_conv_geom* g,
                        const sae_conv_epilogue* epi, int impl, void* stream, const char* who,
                        void* ws = nullptr, int64_t* ws_bytes = nullptr) {
    int rc = validate_geom(g, who);
    if (rc) return rc;
    const bool det = ws_bytes != nullptr;
    bool query = false;
    if (g->N == 0) return det ? det_workspace(ws, ws_bytes, 0, who, &query) : SAE_OK;
    if (!x || !w || !y) return fail(SAE_E_INVALID, "%s: null pointer", who);
    cudaStream_t st = (cudaStream_t)stream;
    EpiParams e = make_epi(epi);
    const bool tc_ok = (det || tc_available()) && tc_fprop_eligible(g);
    if (impl == 2 && !tc_ok) return fail(SAE_E_UNSUPPORTED, "%s: shape not eligible for the wgmma kernel", who);
    if (impl != 1 && tc_ok) {
        if (det && ((rc = det_workspace(ws, ws_bytes, 0, who, &query)) || query)) return rc;
        return tc_fprop(x, w, y, g, e, st, w_lo);
    }
    GatherParams p;
    p.N = g->N; p.OH = g->P; p.OW = g->Q; p.IH = g->H; p.IW = g->W; p.Cs = g->C; p.R = g->R; p.S = g->S;
    p.SY = g->stride; p.DY = 1; p.OFFY = -g->pad_t; p.OFFX = -g->pad_l; p.DIV = 1;
    p.Ncol = g->K; p.K = g->R * g->S * g->C; p.M = (int64_t)g->N * g->P * g->Q;
    if (det) return conv_gather_dispatch_det(x, w, y, p, e, st, w_lo, ws, ws_bytes, who);
    return conv_gather_dispatch(x, w, y, p, e, st, w_lo);
}

static int conv2d_dgrad(const float* dy, const float* wt, const float* wt_lo, float* dx, const sae_conv_geom* g,
                        const sae_conv_epilogue* epi, int impl, void* stream, const char* who,
                        void* ws = nullptr, int64_t* ws_bytes = nullptr) {
    int rc = validate_geom(g, who);
    if (rc) return rc;
    const bool det = ws_bytes != nullptr;
    bool query = false;
    if (g->N == 0) return det ? det_workspace(ws, ws_bytes, 0, who, &query) : SAE_OK;
    if (!dy || !wt || !dx) return fail(SAE_E_INVALID, "%s: null pointer", who);
    cudaStream_t st = (cudaStream_t)stream;
    EpiParams e = make_epi(epi);
    const bool tc_ok = (det || tc_available()) && tc_dgrad_eligible(g);
    if (impl == 2 && !tc_ok) return fail(SAE_E_UNSUPPORTED, "%s: shape not eligible for the wgmma kernel", who);
    if (impl != 1 && tc_ok) {
        if (det && ((rc = det_workspace(ws, ws_bytes, 0, who, &query)) || query)) return rc;
        return tc_dgrad(dy, wt, dx, g, e, st, wt_lo);
    }
    GatherParams p;
    p.N = g->N; p.OH = g->H; p.OW = g->W; p.IH = g->P; p.IW = g->Q; p.Cs = g->K; p.R = g->R; p.S = g->S;
    p.SY = 1; p.DY = -1; p.OFFY = g->pad_t; p.OFFX = g->pad_l; p.DIV = g->stride;
    p.Ncol = g->C; p.K = g->R * g->S * g->K; p.M = (int64_t)g->N * g->H * g->W;
    if (det) return conv_gather_dispatch_det(dy, wt, dx, p, e, st, wt_lo, ws, ws_bytes, who);
    return conv_gather_dispatch(dy, wt, dx, p, e, st, wt_lo);
}

static int conv2d_wgrad(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, void* stream, bool split,
                        const char* who, void* ws = nullptr, int64_t* ws_bytes = nullptr) {
    int rc = validate_geom(g, who);
    if (rc) return rc;
    const bool det = ws_bytes != nullptr;
    bool query = false;
    if (g->N == 0) return det ? det_workspace(ws, ws_bytes, 0, who, &query) : SAE_OK;
    if (!dy || !x || !dw) return fail(SAE_E_INVALID, "%s: null pointer", who);
    cudaStream_t st = (cudaStream_t)stream;
    const bool al = ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x)) & 15) == 0;
    if (impl == 2 && !((det || tc_available()) && al && wgrad_wg_eligible(g)))
        return fail(SAE_E_UNSUPPORTED, "%s: shape not eligible for the wgmma kernel", who);
    if (det) return conv_wgrad_det(dy, x, dw, g, impl, st, split, ws, ws_bytes, who);
    return conv_wgrad(dy, x, dw, g, impl, st, split);
}

extern "C" int sae_conv2d_fprop(const float* x, const float* w, float* y, const sae_conv_geom* g,
                                const sae_conv_epilogue* epi, int impl, void* stream) {
    return conv2d_fprop(x, w, nullptr, y, g, epi, impl, stream, "conv2d_fprop");
}

extern "C" int sae_conv2d_dgrad(const float* dy, const float* wt, float* dx, const sae_conv_geom* g,
                                const sae_conv_epilogue* epi, int impl, void* stream) {
    return conv2d_dgrad(dy, wt, nullptr, dx, g, epi, impl, stream, "conv2d_dgrad");
}

extern "C" int sae_conv2d_wgrad(const float* dy, const float* x, float* dw, const sae_conv_geom* g,
                                int impl, void* stream) {
    return conv2d_wgrad(dy, x, dw, g, impl, stream, false, "conv2d_wgrad");
}

// ---- split-TF32 (fp32-accurate) twins --------------------------------------------------------------------------------------
extern "C" int sae_conv2d_fprop_3xtf32(const float* x, const float* w_hi, const float* w_lo, float* y, const sae_conv_geom* g,
                                       const sae_conv_epilogue* epi, int impl, void* stream) {
    if (!w_lo && g && g->N > 0) return fail(SAE_E_INVALID, "conv2d_fprop_3xtf32: null pointer");
    return conv2d_fprop(x, w_hi, w_lo, y, g, epi, impl, stream, "conv2d_fprop_3xtf32");
}

extern "C" int sae_conv2d_dgrad_3xtf32(const float* dy, const float* wt_hi, const float* wt_lo, float* dx, const sae_conv_geom* g,
                                       const sae_conv_epilogue* epi, int impl, void* stream) {
    if (!wt_lo && g && g->N > 0) return fail(SAE_E_INVALID, "conv2d_dgrad_3xtf32: null pointer");
    return conv2d_dgrad(dy, wt_hi, wt_lo, dx, g, epi, impl, stream, "conv2d_dgrad_3xtf32");
}

extern "C" int sae_conv2d_wgrad_3xtf32(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, void* stream) {
    return conv2d_wgrad(dy, x, dw, g, impl, stream, true, "conv2d_wgrad_3xtf32");
}

// ---- style-modulated convolution with per-sample filters (no modulated copy of the activation) --------------------------
extern "C" int sae_conv2d_query_modulated(const sae_conv_geom* g) {
    if (validate_geom(g, "query_modulated") != SAE_OK) return 0;
    return (tc_available() && tc_per_sample_eligible(g, 0) && tc_per_sample_eligible(g, 1) && wgrad_modulated_eligible(g)) ? 1 : 0;
}

// dir 0: forward, w [N,K,R,S,C]; dir 1: data gradient, w [N,C,R,S,K].  split: the split-TF32 twin (filter pair (w, w_lo))
static int conv2d_per_sample(int dir, const float* x, const float* w, const float* w_lo, float* y, const sae_conv_geom* g,
                             const sae_conv_epilogue* epi, void* stream, bool split, const char* who) {
    int rc = validate_geom(g, who);
    if (rc) return rc;
    if (g->N == 0) return SAE_OK;
    if (!x || !w || (split && !w_lo) || !y) return fail(SAE_E_INVALID, "%s: null pointer", who);
    if (!tc_available()) return fail(SAE_E_UNSUPPORTED, "%s: needs the wgmma path", who);
    return tc_conv_per_sample(x, w, y, g, dir, make_epi(epi), (cudaStream_t)stream, w_lo);
}

// det: the deterministic twin (workspace protocol of det_workspace, which also refuses a null ws_bytes)
static int conv2d_wgrad_modulated(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw, float* ds,
                                  const sae_conv_geom* g, void* stream, bool split, const char* who,
                                  bool det = false, void* ws = nullptr, int64_t* ws_bytes = nullptr) {
    int rc = validate_geom(g, who);
    if (rc) return rc;
    bool query;
    if (g->N == 0) return det ? det_workspace(ws, ws_bytes, 0, who, &query) : SAE_OK;
    if (!dy || !x || !s || !w_krsc || !dw || !ds) return fail(SAE_E_INVALID, "%s: null pointer", who);
    cudaStream_t st = (cudaStream_t)stream;
    if (det) return conv_wgrad_modulated_det(dy, x, s, w_krsc, dw, ds, g, st, split, ws, ws_bytes, who);
    return conv_wgrad_modulated(dy, x, s, w_krsc, dw, ds, g, st, split);
}

extern "C" int sae_conv2d_fprop_per_sample(const float* x, const float* w_nkrsc, float* y, const sae_conv_geom* g,
                                           const sae_conv_epilogue* epi, void* stream) {
    return conv2d_per_sample(0, x, w_nkrsc, nullptr, y, g, epi, stream, false, "conv2d_fprop_per_sample");
}

extern "C" int sae_conv2d_dgrad_per_sample(const float* dy, const float* w_ncrsk, float* dx, const sae_conv_geom* g,
                                           const sae_conv_epilogue* epi, void* stream) {
    return conv2d_per_sample(1, dy, w_ncrsk, nullptr, dx, g, epi, stream, false, "conv2d_dgrad_per_sample");
}

extern "C" int sae_conv2d_wgrad_modulated(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw, float* ds,
                                          const sae_conv_geom* g, void* stream) {
    return conv2d_wgrad_modulated(dy, x, s, w_krsc, dw, ds, g, stream, false, "conv2d_wgrad_modulated");
}

extern "C" int sae_conv2d_fprop_per_sample_3xtf32(const float* x, const float* w_nkrsc_hi, const float* w_nkrsc_lo, float* y,
                                                  const sae_conv_geom* g, const sae_conv_epilogue* epi, void* stream) {
    return conv2d_per_sample(0, x, w_nkrsc_hi, w_nkrsc_lo, y, g, epi, stream, true, "conv2d_fprop_per_sample_3xtf32");
}

extern "C" int sae_conv2d_dgrad_per_sample_3xtf32(const float* dy, const float* w_ncrsk_hi, const float* w_ncrsk_lo, float* dx,
                                                  const sae_conv_geom* g, const sae_conv_epilogue* epi, void* stream) {
    return conv2d_per_sample(1, dy, w_ncrsk_hi, w_ncrsk_lo, dx, g, epi, stream, true, "conv2d_dgrad_per_sample_3xtf32");
}

extern "C" int sae_conv2d_wgrad_modulated_3xtf32(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw,
                                                 float* ds, const sae_conv_geom* g, void* stream) {
    return conv2d_wgrad_modulated(dy, x, s, w_krsc, dw, ds, g, stream, true, "conv2d_wgrad_modulated_3xtf32");
}

// ---- deterministic twins: the arguments of the entry point above, then (workspace, workspace_bytes) --------------------------
extern "C" int sae_conv2d_fprop_det(const float* x, const float* w, float* y, const sae_conv_geom* g, const sae_conv_epilogue* epi,
                                    int impl, void* workspace, int64_t* workspace_bytes, void* stream) {
    if (!workspace_bytes) return fail(SAE_E_INVALID, "conv2d_fprop_det: null workspace_bytes");
    return conv2d_fprop(x, w, nullptr, y, g, epi, impl, stream, "conv2d_fprop_det", workspace, workspace_bytes);
}

extern "C" int sae_conv2d_dgrad_det(const float* dy, const float* wt, float* dx, const sae_conv_geom* g, const sae_conv_epilogue* epi,
                                    int impl, void* workspace, int64_t* workspace_bytes, void* stream) {
    if (!workspace_bytes) return fail(SAE_E_INVALID, "conv2d_dgrad_det: null workspace_bytes");
    return conv2d_dgrad(dy, wt, nullptr, dx, g, epi, impl, stream, "conv2d_dgrad_det", workspace, workspace_bytes);
}

extern "C" int sae_conv2d_wgrad_det(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl, void* workspace,
                                    int64_t* workspace_bytes, void* stream) {
    if (!workspace_bytes) return fail(SAE_E_INVALID, "conv2d_wgrad_det: null workspace_bytes");
    return conv2d_wgrad(dy, x, dw, g, impl, stream, false, "conv2d_wgrad_det", workspace, workspace_bytes);
}

extern "C" int sae_conv2d_fprop_3xtf32_det(const float* x, const float* w_hi, const float* w_lo, float* y, const sae_conv_geom* g,
                                           const sae_conv_epilogue* epi, int impl, void* workspace, int64_t* workspace_bytes,
                                           void* stream) {
    if (!workspace_bytes) return fail(SAE_E_INVALID, "conv2d_fprop_3xtf32_det: null workspace_bytes");
    if (!w_lo && g && g->N > 0) return fail(SAE_E_INVALID, "conv2d_fprop_3xtf32_det: null pointer");
    return conv2d_fprop(x, w_hi, w_lo, y, g, epi, impl, stream, "conv2d_fprop_3xtf32_det", workspace, workspace_bytes);
}

extern "C" int sae_conv2d_dgrad_3xtf32_det(const float* dy, const float* wt_hi, const float* wt_lo, float* dx, const sae_conv_geom* g,
                                           const sae_conv_epilogue* epi, int impl, void* workspace, int64_t* workspace_bytes,
                                           void* stream) {
    if (!workspace_bytes) return fail(SAE_E_INVALID, "conv2d_dgrad_3xtf32_det: null workspace_bytes");
    if (!wt_lo && g && g->N > 0) return fail(SAE_E_INVALID, "conv2d_dgrad_3xtf32_det: null pointer");
    return conv2d_dgrad(dy, wt_hi, wt_lo, dx, g, epi, impl, stream, "conv2d_dgrad_3xtf32_det", workspace, workspace_bytes);
}

extern "C" int sae_conv2d_wgrad_3xtf32_det(const float* dy, const float* x, float* dw, const sae_conv_geom* g, int impl,
                                           void* workspace, int64_t* workspace_bytes, void* stream) {
    if (!workspace_bytes) return fail(SAE_E_INVALID, "conv2d_wgrad_3xtf32_det: null workspace_bytes");
    return conv2d_wgrad(dy, x, dw, g, impl, stream, true, "conv2d_wgrad_3xtf32_det", workspace, workspace_bytes);
}

extern "C" int sae_conv2d_wgrad_modulated_det(const float* dy, const float* x, const float* s, const float* w_krsc, float* dw,
                                              float* ds, const sae_conv_geom* g, void* workspace, int64_t* workspace_bytes,
                                              void* stream) {
    return conv2d_wgrad_modulated(dy, x, s, w_krsc, dw, ds, g, stream, false, "conv2d_wgrad_modulated_det", true, workspace,
                                  workspace_bytes);
}

extern "C" int sae_conv2d_wgrad_modulated_3xtf32_det(const float* dy, const float* x, const float* s, const float* w_krsc,
                                                     float* dw, float* ds, const sae_conv_geom* g, void* workspace,
                                                     int64_t* workspace_bytes, void* stream) {
    return conv2d_wgrad_modulated(dy, x, s, w_krsc, dw, ds, g, stream, true, "conv2d_wgrad_modulated_3xtf32_det", true,
                                  workspace, workspace_bytes);
}

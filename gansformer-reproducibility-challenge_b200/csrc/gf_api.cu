// gf_api.cu -- the extern "C" surface declared in include/gf_attn.h.
#include <stdarg.h>
#include <string.h>
#include <atomic>
#include "gf_common.cuh"

namespace gf {

static thread_local char g_err[1024] = "";
static thread_local int g_path = GF_PATH_NONE;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void set_path(int path) { g_path = path; }
static thread_local int g_cen_path = GF_PATH_NONE;
void set_centroid_path(int path) { g_cen_path = path; }
static std::atomic<long long> g_launches{0};
void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

// The library is built for sm_90a only: refuse anything else loudly instead of failing at launch.
int check_device() {
  static thread_local int checked_dev = -1;
  int dev = -1;
  GF_CUDA_OK(cudaGetDevice(&dev));
  if (dev == checked_dev) return GF_OK;
  int major = 0, minor = 0;
  GF_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  GF_CUDA_OK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) {
    set_error("libgf_attn is built for sm_90a (H100) only; device %d has compute capability %d.%d", dev, major, minor);
    return GF_ERR_UNSUPPORTED;
  }
  checked_dev = dev;
  return GF_OK;
}

int dropout_args(const gf_attn_postop* post, DropoutArgs* out) {
  out->state = nullptr; out->thr = 0; out->salt = 0; out->scale = 1.f;
  if (!post || post->att_dp == 0.f || !post->dp_state) return GF_OK;
  if (!(post->att_dp > 0.f && post->att_dp < 1.f)) { set_error("postop: att_dp = %g must be in [0, 1)", (double)post->att_dp); return GF_ERR_INVALID; }
  double t = (double)post->att_dp * 4294967296.0 + 0.5;
  out->thr = t >= 4294967295.0 ? 4294967295u : (uint32_t)t;
  if (out->thr == 0) out->thr = 1;
  out->salt = post->dp_salt; out->state = post->dp_state; out->scale = 1.f / (1.f - post->att_dp);
  return GF_OK;
}

__global__ void dropout_mask_kernel(float* __restrict__ mask, DropoutArgs D, long long tokens, int KP) {
  const unsigned long long seed = D.state[0], step = D.state[1];
  const long long total = tokens * (KP / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long tok = i / (KP / 4);
    const int q = (int)(i % (KP / 4));
    float mk[4];
    dropout_mult4(D, seed, step, (uint32_t)tok, q, mk);
    reinterpret_cast<float4*>(mask)[i] = make_float4(mk[0], mk[1], mk[2], mk[3]);
  }
}

static int token_pass(const Layout& L, const gf_attn_desc* d, const float* X, float* Xout, float* att, float* ws,
                      const gf_attn_postop* post, cudaStream_t st) {
  int rc;
  if (post && (post->act < 0 || post->act > 1)) { set_error("postop: act must be 0 (linear) or 1 (lrelu), got %d", post->act); return GF_ERR_INVALID; }
  if (post && (post->in_scale || post->post_scale)) {
    if (d->norm != GF_NORM_LAYER && d->norm != GF_NORM_NONE) { set_error("postop: in_scale/post_scale need norm layer or none"); return GF_ERR_UNSUPPORTED; }
    if ((post->in_scale && (post->in_scale_ld < L.C || (post->in_scale_ld & 3) || ((uintptr_t)post->in_scale & 15))) ||
        (post->post_scale && (post->post_scale_ld < L.C || (post->post_scale_ld & 3) || ((uintptr_t)post->post_scale & 15)))) {
      set_error("postop: scale rows must be 16-byte aligned with ld >= C and ld %% 4 == 0");
      return GF_ERR_INVALID;
    }
  }
  if ((rc = norm_stats(L, d, X, ws, st))) return rc;
  const bool tc = !(d->flags & GF_FLAG_FP32_EXACT) && tc_supported(L, d);
  if (post && (post->rgb_out || post->rgb_w)) {
    if (!post->rgb_out || !post->rgb_w || ((uintptr_t)post->rgb_w & 15)) { set_error("postop: fused tRGB needs rgb_w (16-byte aligned) and rgb_out"); return GF_ERR_INVALID; }
    if (!tc || (L.C > 256 && L.KP > 16)) {
      set_error("postop: the fused tRGB is served by the tensor-core path with C <= 256, or C = 512 and k <= 16 (see gf_attn_tc_eligible)");
      return GF_ERR_UNSUPPORTED;
    }
  }
  if (tc) return token_pass_tc(L, d, X, Xout, att, ws, post, st);
  return token_pass_simt(L, d, X, Xout, att, ws, post, st);
}

}  // namespace gf

using namespace gf;

extern "C" {

int gf_attn_abi_version(void) { return GF_ATTN_ABI_VERSION; }
const char* gf_last_error(void) { return g_err; }
int gf_attn_last_path(void) { return g_path; }
int gf_attn_last_centroid_path(void) { return g_cen_path; }
long long gf_attn_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int gf_attn_tc_eligible(const gf_attn_desc* desc) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  return (!(desc->flags & GF_FLAG_FP32_EXACT) && tc_supported(L, desc)) ? 1 : 0;
}

int gf_attn_debug_layout(const gf_attn_desc* desc, long long* out, int n) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  const long long v[15] = {(long long)L.w_PART, (long long)L.w_XBAR, L.nsplit_cen, L.KP, (long long)L.w_M, (long long)L.w_Rt2, (long long)L.w_Ct2,
                           (long long)L.w_total, (long long)L.w_Kp, (long long)L.w_Vt, (long long)L.w_Rt, (long long)L.w_Ct, (long long)L.w_CB,
                           (long long)L.w_NSCALE, (long long)L.w_NSHIFT};
  for (int i = 0; i < n && i < 15; ++i) out[i] = v[i];
  return GF_OK;
}

int gf_attn_debug_tc_schedule(const gf_attn_desc* desc, int rule, int* out, int n) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if ((rc = check_device())) return rc;
  int v[4] = {0, 0, 0, 0};
  if ((rc = tc_schedule(L, desc, rule, v))) return rc;
  if (desc->flags & GF_FLAG_FP32_EXACT) v[0] = v[1] = v[2] = v[3] = 0;   // the CUDA-core kernel serves it
  for (int i = 0; i < n && i < 4; ++i) out[i] = v[i];
  return GF_OK;
}

int gf_attn_folded_floats(const gf_attn_desc* desc, size_t* out_floats) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!out_floats) { set_error("null out_floats"); return GF_ERR_INVALID; }
  *out_floats = L.f_total;
  return GF_OK;
}

int gf_attn_workspace_bytes(const gf_attn_desc* desc, size_t* out_bytes) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!out_bytes) { set_error("null out_bytes"); return GF_ERR_INVALID; }
  *out_bytes = L.w_total * sizeof(float);
  return GF_OK;
}

int gf_attn_fold_weights(const gf_attn_desc* desc, const gf_attn_weights* weights, float* folded, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!weights || !folded) { set_error("gf_attn_fold_weights: null pointer"); return GF_ERR_INVALID; }
  if ((rc = check_device())) return rc;
  return fold_weights(L, desc, weights, folded, (cudaStream_t)stream);
}

int gf_attn_prologue(const gf_attn_desc* desc, const float* Y, const float* folded, void* ws, void* stream) {
  return gf_attn_prologue_ex(desc, Y, folded, ws, nullptr, stream);
}

int gf_attn_prologue_ex(const gf_attn_desc* desc, const float* Y, const float* folded, void* ws, const gf_attn_postop* post, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!Y || !folded || !ws) { set_error("gf_attn_prologue: null pointer"); return GF_ERR_INVALID; }
  if (L.duplex) { set_error("gf_attn_prologue: duplex layers build their keys inside gf_attn_duplex_fwd"); return GF_ERR_INVALID; }
  if ((rc = check_device())) return rc;
  return prologue(L, desc, Y, Y, L.D, folded, (float*)ws, (cudaStream_t)stream, post ? post->in_scale : nullptr, post ? post->in_scale_ld : 0);
}

int gf_attn_prologue_batch(int n, const gf_attn_desc* const* descs, const float* const* Y, const float* const* folded, void* const* ws,
                           const gf_attn_postop* const* posts, void* stream) {
  if (n <= 0) return GF_OK;
  if (n > 64) { set_error("gf_attn_prologue_batch: at most 64 layers per call, got %d", n); return GF_ERR_INVALID; }
  if (!descs || !Y || !folded || !ws) { set_error("gf_attn_prologue_batch: null pointer"); return GF_ERR_INVALID; }
  Layout Ls[64];
  float* wsf[64];
  int rc;
  for (int i = 0; i < n; ++i) {
    if (!descs[i] || !Y[i] || !folded[i] || !ws[i]) { set_error("gf_attn_prologue_batch: null pointer in layer %d", i); return GF_ERR_INVALID; }
    if ((rc = make_layout(descs[i], &Ls[i]))) return rc;
    if (descs[i]->flags & GF_FLAG_CENTROIDS_IN) { set_error("gf_attn_prologue_batch: layer %d takes its centroids as input (no pass-A tables to build)", i); return GF_ERR_INVALID; }
    wsf[i] = (float*)ws[i];
  }
  if ((rc = check_device())) return rc;
  return prologue_batch(n, Ls, descs, Y, folded, wsf, posts, (cudaStream_t)stream);
}

int gf_attn_dropout_mask(const gf_attn_desc* desc, float att_dp, uint32_t dp_salt, const unsigned long long* dp_state, float* mask, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!mask || !dp_state) { set_error("gf_attn_dropout_mask: null pointer"); return GF_ERR_INVALID; }
  gf_attn_postop post;
  memset(&post, 0, sizeof(post));
  post.att_dp = att_dp; post.dp_salt = dp_salt; post.dp_state = dp_state;
  DropoutArgs D;
  if ((rc = dropout_args(&post, &D))) return rc;
  if (!D.thr) { set_error("gf_attn_dropout_mask: att_dp must be > 0"); return GF_ERR_INVALID; }
  if ((rc = check_device())) return rc;
  const long long tokens = (long long)L.B * L.n;
  long long blocks = (tokens * (L.KP / 4) + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  dropout_mask_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(mask, D, tokens, L.KP);
  GF_LAUNCH_OK();
  return GF_OK;
}

int gf_attn_norm_stats(const gf_attn_desc* desc, const float* X, void* ws, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !ws) { set_error("gf_attn_norm_stats: null pointer"); return GF_ERR_INVALID; }
  if ((rc = check_device())) return rc;
  return norm_stats(L, desc, X, (float*)ws, (cudaStream_t)stream);
}

int gf_attn_simplex_fwd(const gf_attn_desc* desc, const float* X, float* Xout, float* att, void* ws, void* stream) {
  return gf_attn_simplex_fwd_ex(desc, X, Xout, att, ws, nullptr, stream);
}

int gf_attn_simplex_fwd_ex(const gf_attn_desc* desc, const float* X, float* Xout, float* att, void* ws,
                           const gf_attn_postop* post, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!X || !Xout || !ws) { set_error("gf_attn_simplex_fwd: null pointer"); return GF_ERR_INVALID; }
  if ((rc = check_device())) return rc;
  return token_pass(L, desc, X, Xout, att, (float*)ws, post, (cudaStream_t)stream);
}

int gf_attn_duplex_fwd(const gf_attn_desc* desc, const float* X, const float* Y, const float* folded,
                       float* Xout, float* att, float* centroids_inout, void* ws_, void* stream) {
  return gf_attn_duplex_fwd_ex(desc, X, Y, folded, Xout, att, centroids_inout, ws_, nullptr, stream);
}

int gf_attn_duplex_fwd_ex(const gf_attn_desc* desc, const float* X, const float* Y, const float* folded,
                          float* Xout, float* att, float* centroids_inout, void* ws_, const gf_attn_postop* post, void* stream) {
  Layout L;
  int rc = make_layout(desc, &L);
  if (rc) return rc;
  if (!L.duplex) { set_error("gf_attn_duplex_fwd: desc.duplex is 0"); return GF_ERR_INVALID; }
  if (!X || !Y || !folded || !Xout || !ws_) { set_error("gf_attn_duplex_fwd: null pointer"); return GF_ERR_INVALID; }
  if (!centroids_inout && (desc->flags & (GF_FLAG_CENTROIDS_IN | GF_FLAG_CENTROIDS_INIT))) { set_error("gf_attn_duplex_fwd: GF_FLAG_CENTROIDS_IN / _INIT without centroids"); return GF_ERR_INVALID; }
  if ((desc->flags & GF_FLAG_CENTROIDS_IN) && (desc->flags & GF_FLAG_CENTROIDS_INIT)) { set_error("gf_attn_duplex_fwd: GF_FLAG_CENTROIDS_IN and _INIT are exclusive"); return GF_ERR_INVALID; }
  if ((rc = check_device())) return rc;
  float* ws = (float*)ws_;
  cudaStream_t st = (cudaStream_t)stream;
  const bool cen_in = (desc->flags & GF_FLAG_CENTROIDS_IN) != 0;
  // explicit centroids are needed when the caller asks for them, for further k-means iterations and for g_img2ltnt; otherwise the
  // keys are built straight from the attention-weighted means (one [B*k, C] x [C, C] product less)
  const bool need_cen = centroids_inout != nullptr || L.iters > 1 || L.img2ltnt;
  float* cen = centroids_inout ? centroids_inout : ws + L.w_CEN;
  if (!cen_in) {
    // load-side scale d (x_in = x * d): pass A sees x only through x.M^T and A.x, so d is folded into M and into Xbar
    const float* isc = post ? post->in_scale : nullptr;
    const int isc_ld = post ? post->in_scale_ld : 0;
    const bool cen_init = (desc->flags & GF_FLAG_CENTROIDS_INIT) != 0;      // `iterative`: the first queries come from the carried-in centroids
    if (!cen_init && !(desc->flags & GF_FLAG_TABLES_READY) && (rc = duplex_tables(L, desc, Y, folded, ws, st, isc, isc_ld))) return rc;
    const bool cen_tc = tc_centroid_supported(L, desc);
    for (int it = 0; it < L.iters; ++it) {
      if ((it > 0 || cen_init) && (rc = duplex_tables_from_centroids(L, desc, cen, Y, folded, ws, st, isc, isc_ld))) return rc;   // queries from the centroids
      if (cen_tc) {
        if ((rc = centroid_pass_tc(L, X, ws, st))) return rc;
        if ((rc = centroid_merge(L, ws, st, isc, isc_ld))) return rc;
        set_centroid_path(GF_PATH_WGMMA_TF32);
      } else {
        if ((rc = centroid_pass_simt(L, desc, X, ws, st, isc, isc_ld))) return rc;
        set_centroid_path(GF_PATH_SIMT_FP32);
      }
      // centroids = Xbar @ Wv2_e + bv2
      // (fp32 when the centroids feed further k-means iterations or are carried on: see duplex_tables_from_centroids)
      if (need_cen && (rc = gemm(st, L.B * L.k, L.C, L.C, ws + L.w_XBAR, L.C, false, folded + L.f_WV2, L.C, false, cen, L.C, 1.f,
                                 nullptr, 0, 1, folded + L.f_BV2, cen_tc && L.iters == 1 && !cen_init)))
        return rc;
    }
  }
  const float* Yv = Y;
  if (L.img2ltnt) {
    if ((rc = img2ltnt(L, Y, cen, folded, ws, st))) return rc;
    Yv = ws + L.w_Y2;
  }
  // V^T depends on the latents only: duplex_tables() already built it, unless pass A was skipped or the latents were modulated
  const bool keys_from_cen = cen_in || need_cen;
  if ((rc = prologue(L, desc, Yv, keys_from_cen ? cen : ws + L.w_XBAR, L.C, folded, ws, st, post ? post->in_scale : nullptr,
                     post ? post->in_scale_ld : 0, !keys_from_cen,
                     cen_in || L.img2ltnt || ((desc->flags & GF_FLAG_CENTROIDS_INIT) && !(desc->flags & GF_FLAG_TABLES_READY)))))
    return rc;
  // attention dropout: the token kernels re-add the constants of the control signal as (1 - sum q) * CB, read from ws (the simplex
  // prologue writes it there; the duplex key path does not)
  if (post && post->att_dp != 0.f && post->dp_state)
    GF_CUDA_OK(cudaMemcpyAsync(ws + L.w_CB, folded + L.f_CB, sizeof(float) * L.Cout, cudaMemcpyDeviceToDevice, st));
  return token_pass(L, desc, X, Xout, att, ws, post, st);
}

}  // extern "C"

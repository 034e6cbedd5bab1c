// engine.cu -- host side of libagp.so: context, stream-ordered workspace, the fused "fit"
// (Gram -> blocked right-looking Cholesky with bordered forward solve -> backward solve -> logpdf),
// prediction, sampling, and the extern "C" ABI declared in include/agp.h.
//
// Data layout in HBM (DESIGN.md s3): the factor lives in ONE column-major buffer of
// (n_pad + 128) x n_pad elements, n_pad = N rounded up to 128 with identity padding.  The Gram kernel
// writes the lower triangle directly into it, the Cholesky runs in place (A = L L', L = U'), and the
// extra 128-row "border" tile holds delta' = (Y - m)' so that the panel TRSM + trailing update
// perform the forward substitution v = L^-1 delta for free (up to 128 right-hand sides).
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <functional>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include <nccl.h>

#include "agp.h"
#include "kernels.h"
#include "umma_ozaki.h"

#define TILE AGP_TILE

struct agp_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;  // look-ahead side stream (bulk of the trailing update)
  cudaStream_t stream3 = nullptr;  // strip inverses of the diagonal blocks (needed only by the solves)
  cudaEvent_t ev_s3 = nullptr, ev_fac = nullptr;
  bool s3_dirty = false;
  std::vector<cudaEvent_t> dep_ev;  // dependency events of the look-ahead schedule
  agp_config cfg{};
  std::string err;
  int64_t info = 0;
  int memspace = AGP_MEM_HOST;
  bool out_dev_override = false;  // internal: outputs of the current call are device pointers whatever memspace says
  double timings[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  cudaEvent_t ev[8]{};
  std::vector<cudaEvent_t> prof_ev;  // pairs around every trailing-update launch
  int prof_used = 0;
  int profile = 1;
  int rank = 0, nranks = 1, grid_p = 1, grid_q = 1;
  ncclComm_t nccl = nullptr;
  OzakiWs oz{};            // slice workspace of the int8-slice fp64 path (cached across fits of the same shape)
  OzakiWs oz2{};           // second slice buffer of the pipelined distributed schedule (panel k+1 is sliced while rest(k) runs)
  OzakiWs ozp{};           // slices of the first half of a two-level outer panel (K = half the panel width; cholesky_inplace)
  int64_t oz_rows = 0, oz2_rows = 0, ozp_rows = 0;
  cudaStream_t stream_comm = nullptr;  // panel broadcasts of the pipelined distributed schedule
  int oz_S = 6;             // ozaki_slices: 6 = six 8-bit digits in the factorisation (slice_format), 5, 7, 8 = 7-bit slices
  int oz_chunk = 16;        // bounded-CTA size (tiles) of the rest updates that run beside a higher-priority stream; 0 = persistent
  int oz_S32 = 4;          // slices of the fp32 operands (4 x 7 bits >= the 24-bit significand)
};

// deep copy of an agp_kernel_composite: the launch descriptor (CompositeDesc, passed by value to the kernels) and the
// per-accumulator weights, on the host (`w`, doubles) and on the device (`desc.w`, in the call's element type)
struct CompState {
  CompositeDesc desc{};
  std::vector<double> w;   // 2 * nacc * D: weights, then 1/r, per accumulator
  int64_t grad_len = 5;
  bool owns_w = false;     // desc.w belongs to this state (a handle's copy) rather than to a call's scratch
};

struct agp_post {
  agp_ctx* ctx = nullptr;
  int dtype = AGP_F64;
  int64_t n = 0, n_pad = 0, lda = 0;
  int D = 0;
  void* L = nullptr;      // (n_pad+TILE) x n_pad
  void* Dinv = nullptr;   // nblk x TILE x TILE
  void* Xt = nullptr;     // n_pad x D transformed points
  void* alpha = nullptr;  // n_pad
  void* ard = nullptr;    // D (device) or null
  void* delta = nullptr;  // n_pad: y - m at the valid rows, 0 at padding
  unsigned char* valid = nullptr;  // n_pad row-validity mask; null while the valid rows are [0, n)
  std::vector<std::pair<int64_t, int64_t>> segs;  // (offset, length) of the valid row segments
  agp_kernel k{};
  int mean_kind = 0;
  double mean_c = 0.0;
  double logdet = 0.0;
  // distributed posterior (multi-GPU fit): the factor stays in its block-column-cyclic form (Lloc: lda x nloc*W, block
  // column jo = lj*R + me) until the first operation that needs it whole; post_replicate() then gathers it over NVLink
  // (one ncclBroadcast per block column from its owner) into L / Dinv and every rank holds a regular handle.
  int dist_R = 0, dist_me = 0, dist_G = 0, dist_nloc = 0;
  int64_t dist_W = 0;
  void* Lloc = nullptr;
  void* Dinv_loc = nullptr;
  CompState* comp = nullptr;  // AGP_COMPOSITE: the handle's own descriptor (k.composite is not kept)
};

struct agp_vfe_post {
  agp_ctx* ctx = nullptr;
  int dtype = AGP_F32;
  int64_t m = 0, m_pad = 0, lda = 0;
  int D = 0;
  void* U = nullptr;      // factor of Kzz + jitter   (m_pad+TILE) x m_pad
  void* Udinv = nullptr;
  void* Lam = nullptr;    // factor of A A' + I
  void* Ldinv = nullptr;
  void* Zt = nullptr;     // m_pad x D
  void* m_e = nullptr;    // m_pad
  void* ard = nullptr;
  agp_kernel k{};
  int mean_kind = 0;
  double mean_c = 0.0;
};

namespace {

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }
static inline int64_t env_int64(const char* name, int64_t dflt) {
  const char* v = getenv(name);
  return v ? atoll(v) : dflt;
}

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t _e = (call);                                                              \
    if (_e != cudaSuccess) {                                                              \
      char _b[512];                                                                       \
      snprintf(_b, sizeof(_b), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      ctx->err = _b;                                                                      \
      return AGP_ERR_CUDA;                                                                \
    }                                                                                     \
  } while (0)

#define CKN(call)                                                                         \
  do {                                                                                    \
    ncclResult_t _r = (call);                                                             \
    if (_r != ncclSuccess) {                                                              \
      char _b[512];                                                                       \
      snprintf(_b, sizeof(_b), "%s:%d %s -> %s", __FILE__, __LINE__, #call, ncclGetErrorString(_r)); \
      ctx->err = _b;                                                                      \
      return AGP_ERR_NCCL;                                                                \
    }                                                                                     \
  } while (0)

template <typename T> struct NcclType;
template <> struct NcclType<float> { static constexpr ncclDataType_t v = ncclFloat; };
template <> struct NcclType<double> { static constexpr ncclDataType_t v = ncclDouble; };

struct Scratch {  // stream-ordered allocations freed together
  agp_ctx* ctx;
  std::vector<void*> ptrs;
  explicit Scratch(agp_ctx* c) : ctx(c) {}
  ~Scratch() { for (void* p : ptrs) cudaFreeAsync(p, ctx->stream); }
  cudaError_t alloc(void** p, size_t bytes) {
    if (bytes == 0) bytes = 16;
    cudaError_t e = cudaMallocAsync(p, bytes, ctx->stream);
    if (e == cudaSuccess) ptrs.push_back(*p);
    return e;
  }
  void release(void* p) {  // ownership moves out
    for (auto& q : ptrs) if (q == p) { q = ptrs.back(); ptrs.pop_back(); return; }
  }
};

template <typename T>
int upload(agp_ctx* ctx, Scratch& sc, const void* src, size_t count, bool always_host, T** out) {
  if (!src || count == 0) { *out = nullptr; return AGP_OK; }
  if (!always_host && ctx->memspace == AGP_MEM_DEVICE) { *out = (T*)src; return AGP_OK; }
  void* d = nullptr;
  CK(sc.alloc(&d, count * sizeof(T)));
  CK(cudaMemcpyAsync(d, src, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  *out = (T*)d;
  return AGP_OK;
}

template <typename T>
int download(agp_ctx* ctx, void* dst, const T* src, size_t count, bool always_host) {
  if (!dst || count == 0) return AGP_OK;
  cudaMemcpyKind kind = (!always_host && (ctx->memspace == AGP_MEM_DEVICE || ctx->out_dev_override)) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  CK(cudaMemcpyAsync(dst, src, count * sizeof(T), kind, ctx->stream));
  return AGP_OK;
}

int check_kernel(agp_ctx* ctx, const agp_kernel* k, int D) {
  if (!k) { ctx->err = "kernel spec is NULL"; return AGP_ERR_INVALID; }
  if (k->family == AGP_COMPOSITE) {  // the descriptor itself is checked by comp_build
    if (ctx->nccl) { ctx->err = "composite kernels are supported on a single-GPU context only"; return AGP_ERR_UNSUPPORTED; }
    // the points are prepared with the top-level transform before the descriptor is read: reject it here, before any
    // upload or launch (a composite carries its transforms in its factors)
    if (k->transform != AGP_T_NONE || k->variance != 1.0) {
      ctx->err = "a composite kernel takes transform AGP_T_NONE and variance 1 (scalings belong to the terms)";
      return AGP_ERR_INVALID;
    }
    if (D <= 0) { ctx->err = "D must be positive"; return AGP_ERR_DIM_MISMATCH; }
    return AGP_OK;
  }
  if (k->family < AGP_SE || k->family > AGP_LINEAR) { ctx->err = "unsupported kernel family"; return AGP_ERR_UNSUPPORTED; }
  if (k->transform < AGP_T_NONE || k->transform > AGP_T_ARD) { ctx->err = "unsupported transform"; return AGP_ERR_UNSUPPORTED; }
  if (k->transform == AGP_T_ARD && !k->ard) { ctx->err = "ARD transform without weights"; return AGP_ERR_INVALID; }
  if (D <= 0) { ctx->err = "D must be positive"; return AGP_ERR_DIM_MISMATCH; }
  return AGP_OK;
}

// Validate an AGP_COMPOSITE kernel and flatten it into a CompState (host side; T = the call's element type, used to read
// the ARD and r arrays).  Accumulators: every stationary / RQ / White factor with no transform or a Scale transform shares
// ONE raw squared distance (d2 = s^2 raw), every such Linear factor one raw dot product; each ARD factor and each Periodic
// factor has its own weighted sum.  Gradient slots follow the layout documented at agp_post_logpdf_grad.
template <typename T>
int comp_build(agp_ctx* ctx, const agp_kernel* k, int D, CompState* cs) {
  const agp_kernel_composite* c = k->composite;
  if (!c || !c->nfactors || !c->variance || !c->factors) { ctx->err = "composite kernel without its descriptor"; return AGP_ERR_INVALID; }
  if (k->transform != AGP_T_NONE || k->variance != 1.0) {
    ctx->err = "a composite kernel takes transform AGP_T_NONE and variance 1 (scalings belong to the terms)";
    return AGP_ERR_INVALID;
  }
  if (c->nterms < 1 || c->nterms > AGP_COMP_MAX) { ctx->err = "composite kernel: 1..8 terms"; return AGP_ERR_INVALID; }
  int nf = 0;
  for (int t = 0; t < c->nterms; ++t) {
    if (c->nfactors[t] < 1) { ctx->err = "composite kernel: every term needs at least one factor"; return AGP_ERR_INVALID; }
    nf += c->nfactors[t];
    if (nf > AGP_COMP_MAX) { ctx->err = "composite kernel: at most 8 factors in all"; return AGP_ERR_INVALID; }
  }
  CompositeDesc& d = cs->desc;
  d = CompositeDesc{};
  d.nterms = c->nterms;
  d.nfactors = nf;
  cs->w.clear();
  int raw_sq = -1, raw_dot = -1;
  auto new_acc = [&](int kind) {
    const int a = d.nacc++;
    d.acc_kind[a] = kind;
    cs->w.resize((size_t)2 * d.nacc * D, 0.0);
    for (int i = 0; i < D; ++i) cs->w[(size_t)2 * a * D + i] = 1.0;
    return a;
  };
  int64_t slot = 5;
  int f = 0;
  for (int t = 0; t < c->nterms; ++t) {
    d.variance[t] = c->variance[t];
    d.g_var[t] = (int)slot++;
    for (int j = 0; j < c->nfactors[t]; ++j, ++f) {
      const agp_kernel_factor& in = c->factors[f];
      CompFactor& F = d.f[f];
      F.family = in.family; F.transform = in.transform; F.term = t;
      F.s = in.transform == AGP_T_SCALE ? in.scale : 1.0;
      F.s2 = 1.0; F.param = in.param;
      F.g_s = F.g_p = F.g_w = F.g_r = -1;
      if (in.family < AGP_SE || in.family > AGP_CONSTANT) { ctx->err = "composite kernel: unsupported factor family"; return AGP_ERR_UNSUPPORTED; }
      if (in.transform < AGP_T_NONE || in.transform > AGP_T_ARD) { ctx->err = "composite kernel: unsupported factor transform"; return AGP_ERR_UNSUPPORTED; }
      if (in.transform == AGP_T_ARD && !in.ard) { ctx->err = "composite kernel: ARD factor without weights"; return AGP_ERR_INVALID; }
      if (in.family == AGP_RQ && !(in.param > 0.0)) { ctx->err = "composite kernel: RationalQuadratic alpha must be > 0"; return AGP_ERR_INVALID; }
      const T* ard = (const T*)in.ard;
      if (in.family == AGP_CONSTANT) {
        F.acc = -1;
      } else if (in.family == AGP_PERIODIC) {
        F.acc = new_acc(COMP_ACC_PER);
        for (int i = 0; i < D; ++i) {
          const double r = in.r ? (double)((const T*)in.r)[i] : 1.0;
          if (!(r > 0.0)) { ctx->err = "composite kernel: Periodic r must be > 0"; return AGP_ERR_INVALID; }
          cs->w[(size_t)2 * F.acc * D + i] = in.transform == AGP_T_ARD ? (double)ard[i] : F.s;
          cs->w[(size_t)(2 * F.acc + 1) * D + i] = 1.0 / r;
        }
      } else if (in.transform == AGP_T_ARD) {
        F.acc = new_acc(in.family == AGP_LINEAR ? COMP_ACC_DOT : COMP_ACC_SQ);
        for (int i = 0; i < D; ++i) cs->w[(size_t)2 * F.acc * D + i] = (double)ard[i];
      } else if (in.family == AGP_LINEAR) {
        if (raw_dot < 0) raw_dot = new_acc(COMP_ACC_DOT);
        F.acc = raw_dot;
        F.s2 = F.s * F.s;
      } else {
        if (raw_sq < 0) raw_sq = new_acc(COMP_ACC_SQ);
        F.acc = raw_sq;
        F.s2 = F.s * F.s;
      }
      if (in.transform == AGP_T_SCALE) F.g_s = (int)slot++;
      else if (in.transform == AGP_T_ARD) { F.g_w = (int)slot; slot += D; }
      if (in.family == AGP_RQ || in.family == AGP_LINEAR || in.family == AGP_CONSTANT) F.g_p = (int)slot++;
      if (in.family == AGP_PERIODIC) { F.g_r = (int)slot; slot += D; }
    }
  }
  if (d.nacc == 0) new_acc(COMP_ACC_SQ);  // Constant factors only: the kernels still carry one (unused) accumulator
  cs->grad_len = slot;
  return AGP_OK;
}

// the descriptor's weights on the device in the element type T: in the call's scratch, or owned by the state (handles)
template <typename T>
int comp_upload(agp_ctx* ctx, Scratch& sc, CompState* cs, bool own) {
  std::vector<T> h(cs->w.begin(), cs->w.end());
  void* dv = nullptr;
  const size_t bytes = h.size() * sizeof(T);
  if (own) CK(cudaMallocAsync(&dv, bytes, ctx->stream));
  else CK(sc.alloc(&dv, bytes));
  CK(cudaMemcpyAsync(dv, h.data(), bytes, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));  // h is a local
  cs->desc.w = dv;
  cs->owns_w = own;
  return AGP_OK;
}

void comp_free(CompState* cs, cudaStream_t s) {
  if (!cs) return;
  if (cs->owns_w && cs->desc.w) cudaFreeAsync((void*)cs->desc.w, s);
  delete cs;
}

void prof_begin(agp_ctx* ctx) { ctx->prof_used = 0; }
cudaEvent_t prof_event(agp_ctx* ctx) {
  if (ctx->prof_used == (int)ctx->prof_ev.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    ctx->prof_ev.push_back(e);
  }
  return ctx->prof_ev[ctx->prof_used++];
}
double prof_total_ms(agp_ctx* ctx) {
  double t = 0;
  for (int i = 0; i + 1 < ctx->prof_used; i += 2) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ctx->prof_ev[i], ctx->prof_ev[i + 1]) == cudaSuccess) t += ms;
  }
  return t;
}

// ---- blocked right-looking Cholesky, in place, lower; rows include the border tile -------------
// Look-ahead (depth 1): after the panel solve of step k, the main stream updates only the NEXT panel
// column and immediately factors / solves panel k+1, while the side stream applies panel k to the rest
// of the trailing matrix.  Event edges: rest_k waits trsm_k; next-column update of step k+1 waits
// rest_k (both touch column block k+2).
static cudaEvent_t dep_event(agp_ctx* ctx, size_t i) {
  while (ctx->dep_ev.size() <= i) {
    cudaEvent_t e;
    cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    ctx->dep_ev.push_back(e);
  }
  return ctx->dep_ev[i];
}

// Two-level blocking: an OUTER panel is G inner blocks (G*128 columns).  Inside it, each inner step is
// potrf -> panel TRSM -> rank-128 update of the remaining inner columns only; the trailing matrix then
// receives ONE rank-(G*128) update per outer panel (K = G*128 halves/quarters the read-modify-write
// passes over C and is what the tensor-core trailing kernels need to be compute-bound).
template <typename T>
void trailing_update(agp_ctx* ctx, T* L, int64_t lda, int64_t row0, int64_t col0, int64_t kcol0, int64_t K,
                     int64_t M, int64_t N, cudaStream_t st, const OzakiWs* oz = nullptr, int64_t oz_row0 = 0) {
  // C = L[row0.., col0..] (M x N, diagonal-anchored iff row0 == col0) -= L[row0.., kcol0..] * L[col0.., kcol0..]'
  if (M <= 0 || N <= 0) return;
  if (ctx->profile) cudaEventRecord(prof_event(ctx), st);
  bool done = false;
  if (oz) {  // int8-sliced tensor-core path: the slices of panel rows [oz_row0, ...) are already in *oz
    if constexpr (std::is_same<T, double>::value) {
      done = ozaki_syrk(*oz, L + row0 + col0 * lda, lda, M, N, 1, 0, 0, col0 - oz_row0, row0 - oz_row0, st) == 0;
    } else {
      done = ozaki_update_ex(*oz, L + row0 + col0 * lda, 1, lda, M, N, 0, -1.0, 0, 0, col0 - oz_row0, row0 - oz_row0, st) == 0;
    }
  }
  if (!done) {
    GemmArgs u{};
    u.A = L + row0 + kcol0 * lda; u.lda = lda;
    u.B = L + row0 + kcol0 * lda; u.ldb = lda;  // column n reads panel row row0 + n, or col0 + n through the map
    u.C = L + row0 + col0 * lda; u.ldc = lda;
    u.M = M; u.N = N; u.K = K; u.alpha_neg = 1; u.beta_one = 1; u.lower_only = 1;
    if (row0 != col0) { u.b_tile_stride = TILE; u.b_off = col0 - row0; }  // lower-only test relative to row0
    launch_gemm<T>(u, st);
  }
  if (ctx->profile) cudaEventRecord(prof_event(ctx), st);
}

// the strip inverses run on stream3; every consumer of Dinv on the main stream joins them first
static void join_inverses(agp_ctx* ctx) {
  if (!ctx->s3_dirty) return;
  cudaEventRecord(ctx->ev_s3, ctx->stream3);
  cudaStreamWaitEvent(ctx->stream, ctx->ev_s3, 0);
  ctx->s3_dirty = false;
}

// resolve the outer panel width (in 128-blocks) and the fp64 trailing-update engine for a problem size:
// explicit config / env wins; "auto" = int8-sliced tensor-core path with 512-wide panels from n_pad >= 8192 (the
// single-GPU fp64 factorisation on eight-bit slices widens them to 1024 from AUTO_NB1024_MIN, see cholesky_inplace)
static int resolve_G(const agp_ctx* ctx, int64_t n_pad) {
  int nb = ctx->cfg.tile_nb;
  if (nb <= 0) nb = (n_pad >= 8192) ? 512 : TILE;
  int G = nb / TILE;
  if (G > 8) G = 8;  // kernels that stage a whole outer block (distributed backward solve) hold at most 8 inner blocks
  return G < 1 ? 1 : G;
}
constexpr int64_t AUTO_NB1024_MIN = 32768;  // C4h (N = 32 768) and C4 (65 536) measured faster at 1024; smaller N not measured
static int resolve_fp64_mode(const agp_ctx* ctx, int64_t n_pad) {
  if (ctx->cfg.fp64_mode >= 0) return ctx->cfg.fp64_mode;
  return n_pad >= 8192 ? 1 : 0;
}
// fp32: 0 = FFMA tile kernels, 1 = int8-sliced tensor-core path (4 slices); auto = int8 slices from n_pad >= 4096
static int resolve_fp32_mode(const agp_ctx* ctx, int64_t n_pad) {
  if (ctx->cfg.fp32_mode >= 0) return ctx->cfg.fp32_mode;
  return n_pad >= 4096 ? 1 : 0;
}
template <typename T> static int resolve_tensor_mode(const agp_ctx* ctx, int64_t n_pad) {
  return std::is_same<T, double>::value ? resolve_fp64_mode(ctx, n_pad) : resolve_fp32_mode(ctx, n_pad);
}
// slice format of a product with K-byte slice rows: fp64 operands follow ozaki_slices -- 6: six 8-bit digits for the
// trailing updates of the Cholesky factorisation (K = panel width <= OZ8_MAX_K, where the int32 accumulators stay exact)
// and seven 7-bit slices for every other product; 5, 7, 8: that many 7-bit slices.  The substitutions and the VFE
// products keep the 7-bit format because their results are used directly and are held to the tile-GEMM path at 1e-8,
// which the 8-bit bound (about 6x the 7-bit one) does not meet after C^-1 amplifies it.  fp32 operands take oz_S32
// 7-bit slices.
struct OzFmt { int S, bits; };
template <typename T> static OzFmt slice_format(const agp_ctx* ctx, int64_t K, bool factor) {
  if (!std::is_same<T, double>::value) return {ctx->oz_S32, 7};
  if (ctx->oz_S == 6) return (factor && K <= OZ8_MAX_K) ? OzFmt{6, 8} : OzFmt{7, 7};
  return {ctx->oz_S, 7};
}
// (re)size a cached slice workspace: rows x K bytes per slice in format f.  The requested format, not ozaki_slices, is
// compared, so a long-K product that falls back to 7-bit slices keeps its workspace from call to call.
static bool ensure_ws(OzakiWs& ws, int64_t& ws_rows, int64_t rows, int K, OzFmt f, cudaStream_t s) {
  if (!ws.SL || ws.K != K || ws_rows < rows || ws.S != f.S || ws.bits != f.bits) {
    if (ws.SL) ozaki_ws_destroy(&ws, s);
    if (ozaki_ws_create(&ws, rows, K, f.S, s, f.bits) == 0) ws_rows = rows;
    else { memset(&ws, 0, sizeof(ws)); ws_rows = 0; }
  }
  return ws.SL != nullptr;
}
// factor: the workspace serves the Cholesky's trailing updates (see slice_format)
template <typename T> static bool ensure_oz2(agp_ctx* ctx, int64_t rows, int K, bool factor, cudaStream_t s) {  // second cached workspace (long-K products)
  return ensure_ws(ctx->oz2, ctx->oz2_rows, rows, K, slice_format<T>(ctx, K, factor), s);
}
template <typename T> static bool ensure_oz(agp_ctx* ctx, int64_t rows, int K, bool factor, cudaStream_t s) {
  return ensure_ws(ctx->oz, ctx->oz_rows, rows, K, slice_format<T>(ctx, K, factor), s);
}

// the route of one panel step: the fp64 split kernels (AGP_POTRF_SPLIT, default on) solve a panel of fewer than
// AGP_TRSM_GEMM_MIN rows below the block by substitution, a taller one by the strip inverse and one in-place GEMM
template <typename T>
int panel_route(int64_t rows_below) {
  if (!std::is_same<T, double>::value || !potrf_split_enabled()) return AGP_PANEL_FUSED;
  static const int64_t trsm_gemm_min = env_int64("AGP_TRSM_GEMM_MIN", 8192);
  return rows_below >= trsm_gemm_min ? AGP_PANEL_SPLIT_GEMM : AGP_PANEL_SPLIT_SUBST;
}

// factor the 128 x 128 block at Akk in place and solve the rows_below panel rows under it, A21 <- A21 L11^-T, by `route`;
// Dinv_k receives inv(L11).  The substitution route leaves the inverse on stream3 (joined by join_inverses).
template <typename T>
void panel_block(agp_ctx* ctx, int route, T* Akk, int64_t lda, int64_t rows_below, T* Dinv_k, double* logdet_part,
                 int blk, int* info, cudaStream_t s) {
  if constexpr (std::is_same<T, double>::value) {
    if (route == AGP_PANEL_SPLIT_SUBST) {
      // short panels (latency-bound): factor on the main stream; the inverse (only the solves need it) on stream3;
      // the panel TRSM by blocked substitution straight from L11
      launch_potrf_factor_f64(Akk, lda, logdet_part, blk, info, s);
      cudaEventRecord(ctx->ev_fac, s);
      cudaStreamWaitEvent(ctx->stream3, ctx->ev_fac, 0);
      launch_trtri_f64(Akk, lda, Dinv_k, ctx->stream3);
      ctx->s3_dirty = true;
      if (rows_below > 0) launch_trsm_sub_f64(Akk + TILE, lda, rows_below, Akk, s);
      return;
    }
    if (route == AGP_PANEL_SPLIT_GEMM) {
      // tall panels: the substitution kernel (32 rows per CTA, 16 dependent steps) runs at ~4 TFLOP/s; the 128x128
      // inverse (8 CTAs, 14 us) followed by ONE in-place DMMA GEMM A21 <- A21 inv(L11)' is ~3x faster from ~8k rows
      launch_potrf_factor_f64(Akk, lda, logdet_part, blk, info, s);
      launch_trtri_f64(Akk, lda, Dinv_k, s);
    }
  }
  if (route == AGP_PANEL_FUSED) launch_potrf_diag<T>(Akk, lda, Dinv_k, logdet_part, blk, info, s);
  if (rows_below > 0) {
    GemmArgs t{};  // A21 <- A21 * inv(L11)'
    t.A = Akk + TILE; t.lda = lda; t.B = Dinv_k; t.ldb = TILE;
    t.C = Akk + TILE; t.ldc = lda; t.M = rows_below; t.N = TILE; t.K = TILE;
    launch_gemm<T>(t, s);
  }
}

// factor one outer panel in place: Lp points at its diagonal element; Gp inner 128-blocks; rows = rows from the
// panel's first row to the end of the (local) column storage (border rows included)
template <typename T>
void factor_panel_step(agp_ctx* ctx, T* Lp, int64_t lda, int Gp, int g, int64_t rows, T* Dinv_p, double* logdet_part,
                       int blk_base, int* info, cudaStream_t s) {
  T* Akk = Lp + (int64_t)g * TILE + (int64_t)g * TILE * lda;
  const int64_t rows_below = rows - (int64_t)(g + 1) * TILE;
  panel_block<T>(ctx, panel_route<T>(rows_below), Akk, lda, rows_below, Dinv_p + (int64_t)g * TILE * TILE, logdet_part,
                 blk_base + g, info, s);
  if (rows_below <= 0) return;
  const int64_t ncols_in = (int64_t)(Gp - (g + 1)) * TILE;  // rank-128 update of the remaining inner columns
  if (ncols_in > 0) {
    GemmArgs u{};
    u.A = Akk + TILE; u.lda = lda; u.B = Akk + TILE; u.ldb = lda;
    u.C = Akk + TILE + (int64_t)TILE * lda; u.ldc = lda;
    u.M = rows_below; u.N = ncols_in; u.K = TILE; u.alpha_neg = 1; u.beta_one = 1; u.lower_only = 1;
    launch_gemm<T>(u, s);
  }
}

// factor one outer panel in place (all inner blocks)
template <typename T>
void factor_panel(agp_ctx* ctx, T* Lp, int64_t lda, int Gp, int64_t rows, T* Dinv_p, double* logdet_part, int blk_base,
                  int* info, cudaStream_t s) {
  for (int g = 0; g < Gp; ++g) factor_panel_step<T>(ctx, Lp, lda, Gp, g, rows, Dinv_p, logdet_part, blk_base, info, s);
}

// factor the outer panel of inner blocks [ko, ko + Gp) of the Cholesky at L.  With `ozp` (slices of K = Gp/2 inner
// blocks) the panel is two-level: factor its first half, apply that half's rank-K update to the second half's columns
// (every row below the first half: a rectangle plus the lower tiles of its diagonal block) on the int8-slice kernel,
// then factor the second half.  The rank-128 DMMA updates inside each half then span at most Gp/2 - 1 inner blocks, as
// in a panel of half the width, instead of Gp - 1.
template <typename T>
void factor_outer_panel(agp_ctx* ctx, T* L, int64_t lda, int ko, int Gp, int64_t rows_total, T* Dinv,
                        double* logdet_part, int* info, cudaStream_t s, const OzakiWs* ozp) {
  const int64_t p0 = (int64_t)ko * TILE;
  if (!ozp || (int64_t)Gp * TILE != 2 * (int64_t)ozp->K) {
    factor_panel<T>(ctx, L + p0 + p0 * lda, lda, Gp, rows_total - p0, Dinv + p0 * TILE, logdet_part, ko, info, s);
    return;
  }
  const int h = Gp / 2;
  const int64_t h0 = p0 + (int64_t)h * TILE;  // first row / column of the second half
  factor_panel<T>(ctx, L + p0 + p0 * lda, lda, h, rows_total - p0, Dinv + p0 * TILE, logdet_part, ko, info, s);
  constexpr int is_f32 = std::is_same<T, double>::value ? 0 : 1;
  ozaki_prepare_ex(*ozp, L + h0 + p0 * lda, is_f32, 0, lda, rows_total - h0, 0, s);
  trailing_update<T>(ctx, L, lda, h0, h0, p0, ozp->K, rows_total - h0, (int64_t)(Gp - h) * TILE, s, ozp, h0);
  factor_panel<T>(ctx, L + h0 + h0 * lda, lda, Gp - h, rows_total - h0, Dinv + h0 * TILE, logdet_part, ko + h, info, s);
}

template <typename T>
void cholesky_inplace(agp_ctx* ctx, T* L, int64_t lda, int64_t n_pad, int64_t rows_total, T* Dinv,
                      double* logdet_part, int* info) {
  cudaStream_t s = ctx->stream, s2 = ctx->stream2;
  const int nblk = (int)(n_pad / TILE);
  const int fp64_mode = resolve_tensor_mode<T>(ctx, n_pad);  // 1: int8-sliced tensor-core trailing update (fp64: slice_format, fp32: 4 slices)
  int G = resolve_G(ctx, n_pad);
  if (!std::is_same<T, double>::value && fp64_mode == 1 && ctx->cfg.tile_nb <= 0 && n_pad >= 4096) G = 4;  // 512-wide panels
  // fp64 on eight-bit slices: 1024-wide (two-level) panels from AUTO_NB1024_MIN, where they measured faster (DESIGN §6)
  if (std::is_same<T, double>::value && fp64_mode == 1 && ctx->cfg.tile_nb <= 0 && ctx->oz_S == 6 &&
      n_pad >= AUTO_NB1024_MIN)
    G = 8;
  const bool oz_ok = fp64_mode == 1 && nblk > 2 * G && ensure_oz<T>(ctx, rows_total, G * TILE, true, s) &&
                     (std::is_same<T, double>::value || ctx->oz.bulk == 2);
  // two-level outer panels (factor_outer_panel) where the trailing update runs on eight-bit slices and the panel is wider
  // than 512; the in-panel slices keep their own workspace, so neither it nor the trailing one is recreated per panel
  const OzakiWs* ozp = nullptr;
  if (oz_ok && ctx->oz.bits == 8 && G > 4 && G % 2 == 0 &&
      ensure_ws(ctx->ozp, ctx->ozp_rows, rows_total, G / 2 * TILE, slice_format<T>(ctx, G / 2 * TILE, true), s) &&
      ctx->ozp.bits == 8)
    ozp = &ctx->ozp;
  const bool la = ctx->cfg.lookahead != 0 && nblk > 2 * G;
  const bool la2 = la && ctx->cfg.lookahead >= 2;
  bool rest_pending = false, restA_pending = false, last_rest_full = false;
  size_t ev_idx = 0, last_rest = 0, last_restA = 0;
  for (int ko = 0; ko < nblk; ko += G) {
    const int g_end = (ko + G < nblk) ? ko + G : nblk;  // inner blocks [ko, g_end)
    factor_outer_panel<T>(ctx, L, lda, ko, g_end - ko, rows_total, Dinv, logdet_part, info, s, ozp);
    const int64_t t0 = (int64_t)g_end * TILE;           // first trailing row/column
    const int64_t cols_trail = n_pad - t0;
    if (cols_trail <= 0) continue;
    const int64_t K = (int64_t)(g_end - ko) * TILE, kc0 = (int64_t)ko * TILE;
    const OzakiWs* oz = nullptr;
    // int8-slice path: needs the full outer-panel width it was sized for and enough trailing work to pay for slicing
    if (oz_ok && K == ctx->oz.K && cols_trail >= 2 * TILE) oz = &ctx->oz;
    constexpr int is_f32 = std::is_same<T, double>::value ? 0 : 1;
    if (!la) {
      if (oz) ozaki_prepare_ex(*oz, L + t0 + kc0 * lda, is_f32, 0, lda, rows_total - t0, 0, s);
      trailing_update<T>(ctx, L, lda, t0, t0, kc0, K, rows_total - t0, cols_trail, s, oz, t0);
      continue;
    }
    if (la2 && !oz) {
      // EXPERIMENTAL look-ahead depth 2 (cfg.lookahead = 2 / AGP_LOOKAHEAD=2, DMMA path only -- the int8-slice path would
      // need a second slice buffer; not yet run on a device).  The rest update is split: restA = the panel after next,
      // restB = everything beyond.  The next-panel update of step k+1 needs only restA(k), so the latency-bound chain
      // (potrf -> TRSM -> next-panel update) no longer waits for the bulk of the previous rest update; restB(k) has two
      // chain steps to finish instead of one (it is serialised behind restB(k-1) and restA(k) on the side stream).
      cudaEvent_t e_panel = dep_event(ctx, ev_idx++), e_restA = dep_event(ctx, ev_idx++), e_restB = dep_event(ctx, ev_idx++);
      if (restA_pending) cudaStreamWaitEvent(s, dep_event(ctx, last_restA), 0);
      // a previous step may have used the depth-1 branch (int8-slice panel followed by a short DMMA tail): its rest update
      // on the side stream touches the same block column as the update below
      if (rest_pending && last_rest_full) cudaStreamWaitEvent(s, dep_event(ctx, last_rest), 0);
      cudaEventRecord(e_panel, s);
      const int64_t next_cols = (cols_trail < (int64_t)G * TILE) ? cols_trail : (int64_t)G * TILE;
      trailing_update<T>(ctx, L, lda, t0, t0, kc0, K, rows_total - t0, next_cols, s, nullptr, t0);
      restA_pending = false;
      rest_pending = false;
      if (cols_trail > next_cols) {
        const int64_t r0 = t0 + next_cols;
        const int64_t colsA = (n_pad - r0 < (int64_t)G * TILE) ? (n_pad - r0) : (int64_t)G * TILE;
        cudaStreamWaitEvent(s2, e_panel, 0);
        trailing_update<T>(ctx, L, lda, r0, r0, kc0, K, rows_total - r0, colsA, s2, nullptr, t0);
        cudaEventRecord(e_restA, s2);
        restA_pending = true;
        last_restA = ev_idx - 2;
        const int64_t r1 = r0 + colsA;
        if (n_pad > r1) trailing_update<T>(ctx, L, lda, r1, r1, kc0, K, rows_total - r1, n_pad - r1, s2, nullptr, t0);
        cudaEventRecord(e_restB, s2);
        rest_pending = true;
        last_rest_full = false;  // restB never touches the next panel's columns
        last_rest = ev_idx - 1;
      }
      continue;
    }
    cudaEvent_t e_panel = dep_event(ctx, ev_idx++), e_rest = dep_event(ctx, ev_idx++);
    if (rest_pending) cudaStreamWaitEvent(s, dep_event(ctx, last_rest), 0);  // also frees the slice buffer
    if (restA_pending) { cudaStreamWaitEvent(s, dep_event(ctx, last_restA), 0); restA_pending = false; }
    if (oz) ozaki_prepare_ex(*oz, L + t0 + kc0 * lda, is_f32, 0, lda, rows_total - t0, 0, s);
    cudaEventRecord(e_panel, s);
    const int64_t next_cols = (cols_trail < (int64_t)G * TILE) ? cols_trail : (int64_t)G * TILE;
    trailing_update<T>(ctx, L, lda, t0, t0, kc0, K, rows_total - t0, next_cols, s, oz, t0);  // next outer panel first
    rest_pending = false;
    if (cols_trail > next_cols) {
      const int64_t r0 = t0 + next_cols;
      cudaStreamWaitEvent(s2, e_panel, 0);
      // the panel chain on the (higher-priority) main stream gets SMs between CTAs.  oz_chunk is the area of a bounded CTA
      // at K = 512; a wider panel's tile takes K / 512 times as long, so the CTA takes that many times fewer tiles
      if (oz) oz->chunk_tiles = K > 512 && ctx->oz_chunk > 0 ? std::max(1, (int)(ctx->oz_chunk * 512 / K)) : ctx->oz_chunk;
      trailing_update<T>(ctx, L, lda, r0, r0, kc0, K, rows_total - r0, n_pad - r0, s2, oz, t0);
      if (oz) oz->chunk_tiles = 0;
      cudaEventRecord(e_rest, s2);
      rest_pending = true;
      last_rest_full = true;
      last_rest = ev_idx - 1;
    }
  }
  if (rest_pending) cudaStreamWaitEvent(s, dep_event(ctx, last_rest), 0);
  join_inverses(ctx);  // Dinv (stream3) is complete before any solve on the main stream
}

// V <- L^-1 V on the tensor cores: two-level blocked substitution.  Inside an outer block of W = 512 rows the 128-step
// loop runs on the tile GEMMs (W^2 ncols work); everything below the block receives ONE rank-W update
//   B[below] -= L[below, block] * B[block]
// on the int8-sliced tensor-core kernel: the L panel (rows_below x W, row-contiguous) and B[block]' (ncols x W, k-major) are
// sliced into one workspace (A rows first, B rows behind them) and the product is a rectangular update of B[below].
// This is `C.U' \ X` of /root/reference/src/util/common_covmat_ops.jl:54,90 (prediction, N^2 M flops at config C3) and the
// A = U' \ K_zx solve of /root/reference/src/sparse_approximations.jl:296.
template <typename T>
bool forward_subst_multi_tc(agp_ctx* ctx, const T* L, int64_t lda, const T* Dinv, int64_t n_pad, T* B, int64_t ldb,
                            int64_t ncols) {
  cudaStream_t s = ctx->stream;
  constexpr int GW = 4;
  const int64_t W = (int64_t)GW * TILE;
  const int nblk = (int)(n_pad / TILE);
  constexpr int is_f32 = std::is_same<T, double>::value ? 0 : 1;
  const int64_t a_rows = round_up(n_pad, TILE);
  if (!ensure_oz<T>(ctx, a_rows + ncols, (int)W, false, s) || ctx->oz.bulk != 2) return false;
  const OzakiWs& ws = ctx->oz;
  for (int ko = 0; ko < nblk; ko += GW) {
    const int k_end = (ko + GW < nblk) ? ko + GW : nblk;
    const int64_t blk_end = (int64_t)k_end * TILE;
    for (int k = ko; k < k_end; ++k) {  // in-block substitution (128-steps, rows of this outer block only)
      T* Bk = B + (int64_t)k * TILE;
      GemmArgs a{};
      a.A = Dinv + (int64_t)k * TILE * TILE; a.lda = TILE; a.a_kmajor = 0;
      a.B = Bk; a.ldb = ldb; a.b_kmajor = 1;
      a.C = Bk; a.ldc = ldb; a.M = TILE; a.N = ncols; a.K = TILE;
      launch_gemm<T>(a, s);
      const int64_t rows_in = blk_end - (int64_t)(k + 1) * TILE;
      if (rows_in <= 0) continue;
      GemmArgs u{};
      u.A = L + (int64_t)(k + 1) * TILE + (int64_t)k * TILE * lda; u.lda = lda; u.a_kmajor = 0;
      u.B = Bk; u.ldb = ldb; u.b_kmajor = 1;
      u.C = Bk + TILE; u.ldc = ldb; u.M = rows_in; u.N = ncols; u.K = TILE; u.alpha_neg = 1; u.beta_one = 1;
      launch_gemm<T>(u, s);
    }
    const int64_t rows_below = n_pad - blk_end, Kw = blk_end - (int64_t)ko * TILE;
    if (rows_below <= 0) continue;
    if (Kw != W) {  // ragged last outer block (n_pad not a multiple of 512): finish on the tile GEMM
      GemmArgs u{};
      u.A = L + blk_end + (int64_t)ko * TILE * lda; u.lda = lda; u.a_kmajor = 0;
      u.B = B + (int64_t)ko * TILE; u.ldb = ldb; u.b_kmajor = 1;
      u.C = B + blk_end; u.ldc = ldb; u.M = rows_below; u.N = ncols; u.K = Kw; u.alpha_neg = 1; u.beta_one = 1;
      launch_gemm<T>(u, s);
      continue;
    }
    ozaki_prepare_ex(ws, L + blk_end + (int64_t)ko * TILE * lda, is_f32, 0, lda, rows_below, 0, s);
    ozaki_prepare_ex(ws, B + (int64_t)ko * TILE, is_f32, 1, ldb, ncols, a_rows, s);
    if (ozaki_update_ex(ws, B + blk_end, is_f32, ldb, rows_below, ncols, 1, -1.0, 0, 0, a_rows, 0, s) != 0) return false;
  }
  return true;
}

// V <- L^-1 V for a n_pad x ncols block of right-hand sides (ncols multiple of 4), in place
template <typename T>
void forward_subst_multi(agp_ctx* ctx, const T* L, int64_t lda, const T* Dinv, int64_t n_pad, T* B, int64_t ldb,
                         int64_t ncols) {
  cudaStream_t s = ctx->stream;
  const int nblk = (int)(n_pad / TILE);
  static const int64_t tc_min_cols = env_int64("AGP_SOLVE_TC_MIN_COLS", 512);
  if (resolve_tensor_mode<T>(ctx, n_pad >= 2048 ? (int64_t)1 << 20 : 0) == 1 && n_pad >= 2048 && ncols % TILE == 0 &&
      ncols >= tc_min_cols) {
    if (forward_subst_multi_tc<T>(ctx, L, lda, Dinv, n_pad, B, ldb, ncols)) return;
  }
  for (int k = 0; k < nblk; ++k) {
    T* Bk = B + (int64_t)k * TILE;
    GemmArgs a{};
    a.A = Dinv + (int64_t)k * TILE * TILE; a.lda = TILE; a.a_kmajor = 0;
    a.B = Bk; a.ldb = ldb; a.b_kmajor = 1;
    a.C = Bk; a.ldc = ldb; a.M = TILE; a.N = ncols; a.K = TILE;
    launch_gemm<T>(a, s);
    const int64_t rows_below = n_pad - (int64_t)(k + 1) * TILE;
    if (rows_below <= 0) continue;
    GemmArgs u{};
    u.A = L + (int64_t)(k + 1) * TILE + (int64_t)k * TILE * lda; u.lda = lda; u.a_kmajor = 0;
    u.B = Bk; u.ldb = ldb; u.b_kmajor = 1;
    u.C = Bk + TILE; u.ldc = ldb; u.M = rows_below; u.N = ncols; u.K = TILE; u.alpha_neg = 1; u.beta_one = 1;
    launch_gemm<T>(u, s);
  }
}

// B <- L^-T B: forward_subst_multi's mirror, from the last block to the first.  Block k: B_k = Dinv_k' B_k (Dinv's blocks
// are zero above their diagonal, so the full-block product is the triangular one), then B[above] -= L[block, above]' B_k,
// both on the tile GEMM with the L operand read k-major.  The two-level schedule keeps the forward path's outer blocks
// of 512 rows, visited last to first: the 128-steps stay inside the outer block, and everything above it receives one
// rank-512 update on the int8-sliced kernel, with the L panel (the block's rows, the columns above) sliced k-major.  The
// ragged outer block (n_pad not a multiple of 512, here the first one visited) updates the rows above on the tile GEMM.
template <typename T>
bool backward_subst_multi_tc(agp_ctx* ctx, const T* L, int64_t lda, const T* Dinv, int64_t n_pad, T* B, int64_t ldb,
                             int64_t ncols) {
  cudaStream_t s = ctx->stream;
  constexpr int GW = 4;
  const int64_t W = (int64_t)GW * TILE;
  const int nblk = (int)(n_pad / TILE);
  constexpr int is_f32 = std::is_same<T, double>::value ? 0 : 1;
  const int64_t a_rows = round_up(n_pad, TILE);
  if (!ensure_oz<T>(ctx, a_rows + ncols, (int)W, false, s) || ctx->oz.bulk != 2) return false;
  const OzakiWs& ws = ctx->oz;
  for (int ko = (nblk - 1) / GW * GW; ko >= 0; ko -= GW) {
    const int k_end = (ko + GW < nblk) ? ko + GW : nblk;
    const int64_t blk0 = (int64_t)ko * TILE;
    for (int k = k_end - 1; k >= ko; --k) {  // in-block substitution (128-steps, rows of this outer block only)
      T* Bk = B + (int64_t)k * TILE;
      GemmArgs a{};
      a.A = Dinv + (int64_t)k * TILE * TILE; a.lda = TILE; a.a_kmajor = 1;
      a.B = Bk; a.ldb = ldb; a.b_kmajor = 1;
      a.C = Bk; a.ldc = ldb; a.M = TILE; a.N = ncols; a.K = TILE;
      launch_gemm<T>(a, s);
      const int64_t rows_in = (int64_t)k * TILE - blk0;
      if (rows_in <= 0) continue;
      GemmArgs u{};
      u.A = L + (int64_t)k * TILE + blk0 * lda; u.lda = lda; u.a_kmajor = 1;
      u.B = Bk; u.ldb = ldb; u.b_kmajor = 1;
      u.C = B + blk0; u.ldc = ldb; u.M = rows_in; u.N = ncols; u.K = TILE; u.alpha_neg = 1; u.beta_one = 1;
      launch_gemm<T>(u, s);
    }
    const int64_t rows_above = blk0, Kw = (int64_t)k_end * TILE - blk0;
    if (rows_above <= 0) continue;
    if (Kw != W) {  // ragged outer block: finish on the tile GEMM
      GemmArgs u{};
      u.A = L + blk0; u.lda = lda; u.a_kmajor = 1;
      u.B = B + blk0; u.ldb = ldb; u.b_kmajor = 1;
      u.C = B; u.ldc = ldb; u.M = rows_above; u.N = ncols; u.K = Kw; u.alpha_neg = 1; u.beta_one = 1;
      launch_gemm<T>(u, s);
      continue;
    }
    ozaki_prepare_ex(ws, L + blk0, is_f32, 1, lda, rows_above, 0, s);
    ozaki_prepare_ex(ws, B + blk0, is_f32, 1, ldb, ncols, a_rows, s);
    if (ozaki_update_ex(ws, B, is_f32, ldb, rows_above, ncols, 1, -1.0, 0, 0, a_rows, 0, s) != 0) return false;
  }
  return true;
}

// B <- L^-T B for a n_pad x ncols block of right-hand sides (ncols multiple of 4), in place; the tensor-core schedule
// under forward_subst_multi's rule
template <typename T>
void backward_subst_multi(agp_ctx* ctx, const T* L, int64_t lda, const T* Dinv, int64_t n_pad, T* B, int64_t ldb,
                          int64_t ncols) {
  cudaStream_t s = ctx->stream;
  const int nblk = (int)(n_pad / TILE);
  static const int64_t tc_min_cols = env_int64("AGP_SOLVE_TC_MIN_COLS", 512);
  if (resolve_tensor_mode<T>(ctx, n_pad >= 2048 ? (int64_t)1 << 20 : 0) == 1 && n_pad >= 2048 && ncols % TILE == 0 &&
      ncols >= tc_min_cols) {
    if (backward_subst_multi_tc<T>(ctx, L, lda, Dinv, n_pad, B, ldb, ncols)) return;
  }
  for (int k = nblk - 1; k >= 0; --k) {
    T* Bk = B + (int64_t)k * TILE;
    GemmArgs a{};
    a.A = Dinv + (int64_t)k * TILE * TILE; a.lda = TILE; a.a_kmajor = 1;
    a.B = Bk; a.ldb = ldb; a.b_kmajor = 1;
    a.C = Bk; a.ldc = ldb; a.M = TILE; a.N = ncols; a.K = TILE;
    launch_gemm<T>(a, s);
    const int64_t rows_above = (int64_t)k * TILE;
    if (rows_above <= 0) continue;
    GemmArgs u{};
    u.A = L + (int64_t)k * TILE; u.lda = lda; u.a_kmajor = 1;
    u.B = Bk; u.ldb = ldb; u.b_kmajor = 1;
    u.C = B; u.ldc = ldb; u.M = rows_above; u.N = ncols; u.K = TILE; u.alpha_neg = 1; u.beta_one = 1;
    launch_gemm<T>(u, s);
  }
}

template <typename T>
void fill_gram_params(GramParams& gp, const agp_kernel* k, int symmetric, int lower_only, int64_t va, int64_t vb,
                      const agp_noise* noise, const T* noise_v_dev, const CompState* comp = nullptr) {
  gp.comp = comp ? &comp->desc : nullptr;
  gp.family = k->family;
  gp.variance = k->variance;
  gp.linear_c = k->linear_c;
  gp.symmetric = symmetric;
  gp.lower_only = lower_only;
  gp.valid_a = va;
  gp.valid_b = vb;
  gp.noise_kind = noise ? noise->kind : -1;
  gp.noise_s = noise ? noise->s : 0.0;
  gp.noise_v = noise_v_dev;
}

// transformed, padded, point-major copy of a point set on the device
template <typename T>
int prep_points(agp_ctx* ctx, Scratch& sc, const agp_kernel* k, const T* ard_dev, int layout, const void* X,
                int64_t n, int64_t n_pad, int D, T** Xt_out, bool keep) {
  T* Xd = nullptr;
  int rc = upload<T>(ctx, sc, X, (size_t)n * D, false, &Xd);
  if (rc) return rc;
  void* xt = nullptr;
  CK(cudaMallocAsync(&xt, (size_t)(n_pad > 0 ? n_pad : 1) * D * sizeof(T), ctx->stream));
  if (!keep) sc.ptrs.push_back(xt);
  launch_prep_points<T>(Xd, layout, n, n_pad, D, k->transform, k->scale, ard_dev, (T*)xt, ctx->stream);
  *Xt_out = (T*)xt;
  return AGP_OK;
}

template <typename T>
int fit_impl(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout,
             const void* X, int64_t N, int D, const void* Y, int S, void* logpdf_out, void* alpha_out,
             agp_post** post_out, T** L_keep /*optional raw factor out for rand*/, int64_t* lda_out,
             Scratch* outer_sc) {
  int rc = check_kernel(ctx, k, D);
  if (rc) return rc;
  if (N <= 0) { ctx->err = "N must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (S < 0 || S > TILE) { ctx->err = "number of right-hand sides must be in [0,128]"; return AGP_ERR_UNSUPPORTED; }
  if (S > 0 && !Y) { ctx->err = "Y is NULL"; return AGP_ERR_INVALID; }
  static const agp_mean zero_mean{0, 0.0, nullptr};
  static const agp_noise default_noise{0, 1e-18, nullptr};  // default_sigma^2, finite_gp_projection.jl:17
  if (!mean) mean = &zero_mean;
  if (!noise) noise = &default_noise;
  if (mean->kind == 2 && !mean->v) { ctx->err = "mean vector is NULL"; return AGP_ERR_INVALID; }
  if (noise->kind == 1 && !noise->v) { ctx->err = "noise vector is NULL"; return AGP_ERR_INVALID; }

  CompState comp_local;
  if (k->family == AGP_COMPOSITE) { rc = comp_build<T>(ctx, k, D, &comp_local); if (rc) return rc; }

  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  Scratch sc(ctx);
  const int64_t n_pad = round_up(N, TILE), lda = n_pad + TILE;
  const int nblk = (int)(n_pad / TILE);
  prof_begin(ctx);
  CK(cudaEventRecord(ctx->ev[0], s));

  // the factor is allocated FIRST: the stream-ordered pool then hands back the block the previous fit freed, before the small
  // staging buffers below can split it (a split forces a fresh multi-GB allocation from the OS: 0.1-0.6 s, seen as a
  // sporadic e2e-only slowdown in round 2, tools/dist1_probe.py)
  void* Lv = nullptr;
  CK(cudaMallocAsync(&Lv, (size_t)lda * n_pad * sizeof(T), s));
  struct BufGuard { void* p; cudaStream_t s; ~BufGuard() { if (p) cudaFreeAsync(p, s); } } lguard{Lv, s};  // error returns
  // ---- H2D
  T *ard_d = nullptr, *mean_d = nullptr, *noise_d = nullptr, *Yd = nullptr, *Xt = nullptr;
  if (k->transform == AGP_T_ARD) { rc = upload<T>(ctx, sc, k->ard, D, true, &ard_d); if (rc) return rc; }
  if (mean->kind == 2) { rc = upload<T>(ctx, sc, mean->v, N, true, &mean_d); if (rc) return rc; }
  if (noise->kind == 1) { rc = upload<T>(ctx, sc, noise->v, N, true, &noise_d); if (rc) return rc; }
  if (S > 0) { rc = upload<T>(ctx, sc, Y, (size_t)N * S, false, &Yd); if (rc) return rc; }
  const bool keep = (post_out != nullptr);
  rc = prep_points<T>(ctx, sc, k, ard_d, layout, X, N, n_pad, D, &Xt, keep);
  if (rc) return rc;
  CompState* comp = nullptr;
  if (k->family == AGP_COMPOSITE) {
    comp = keep ? new CompState(comp_local) : &comp_local;
    rc = comp_upload<T>(ctx, sc, comp, keep);
    if (rc) { if (keep) comp_free(comp, s); return rc; }
  }
  struct CompGuard { CompState* c; cudaStream_t s; ~CompGuard() { if (c) comp_free(c, s); } } cguard{keep ? comp : nullptr, s};
  CK(cudaEventRecord(ctx->ev[1], s));

  // ---- buffers
  void *Dinvv = nullptr, *alphav = nullptr;
  lguard.p = nullptr;  // ownership passes to the handle / scratch lists below
  CK(cudaMallocAsync(&Dinvv, (size_t)nblk * TILE * TILE * sizeof(T), s));
  CK(cudaMallocAsync(&alphav, (size_t)n_pad * sizeof(T), s));
  T* L = (T*)Lv; T* Dinv = (T*)Dinvv; T* alpha = (T*)alphav;
  agp_post* post = nullptr;
  struct PostGuard { agp_post* p; ~PostGuard() { if (p) agp_post_free(p); } } pguard{nullptr};  // early error returns
  if (keep) {
    post = new agp_post();
    pguard.p = post;
    post->ctx = ctx; post->dtype = sizeof(T) == 8 ? AGP_F64 : AGP_F32;
    post->n = N; post->n_pad = n_pad; post->lda = lda; post->D = D;
    post->L = Lv; post->Dinv = Dinvv; post->Xt = Xt; post->alpha = alphav;
    post->k = *k; post->k.ard = nullptr; post->k.composite = nullptr;
    post->comp = comp;  // freed with the handle
    cguard.c = nullptr;
    post->mean_kind = mean->kind == 2 ? 0 : mean->kind; post->mean_c = mean->c;
    post->segs.push_back({0, N});
    CK(cudaMallocAsync(&post->delta, (size_t)n_pad * sizeof(T), s));
    if (ard_d) { sc.release(ard_d); post->ard = ard_d; }
  } else if (L_keep) {
    outer_sc->ptrs.push_back(Lv); sc.ptrs.push_back(Dinvv); sc.ptrs.push_back(alphav);
  } else {
    sc.ptrs.push_back(Lv); sc.ptrs.push_back(Dinvv); sc.ptrs.push_back(alphav);
  }
  double* dscal = nullptr;  // [0..nblk) logdet parts, [nblk..nblk+TILE) sqmahal, [+1] logdet
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)(nblk + TILE + 2) * sizeof(double)));
  dscal = (double*)tmp;
  int* dinfo = nullptr;
  CK(sc.alloc(&tmp, sizeof(int)));
  dinfo = (int*)tmp;
  CK(cudaMemsetAsync(dinfo, 0, sizeof(int), s));
  T* rwork = nullptr;
  CK(sc.alloc(&tmp, (size_t)(S > 0 ? S : 1) * n_pad * sizeof(T)));
  rwork = (T*)tmp;
  int* dflags = nullptr;
  CK(sc.alloc(&tmp, (size_t)(nblk + 1) * sizeof(int)));
  dflags = (int*)tmp;
  T* lp_d = nullptr;
  CK(sc.alloc(&tmp, (size_t)TILE * sizeof(T)));
  lp_d = (T*)tmp;

  // ---- Gram (+ noise) straight into the factor buffer, border rows = delta'
  GramParams gp{};
  fill_gram_params<T>(gp, k, 1, 1, N, N, noise, noise_d, comp);
  launch_gram<T>(Xt, Xt, n_pad, n_pad, D, L, lda, gp, s);
  launch_border_init<T>(L, lda, N, n_pad, Yd, N, S, mean->kind, mean->c, mean_d, s);
  if (keep) {
    if (S > 0) launch_extract_v<T>(L, lda, n_pad, 1, (T*)post->delta, dscal + nblk, s);  // delta = border row 0
    else CK(cudaMemsetAsync(post->delta, 0, (size_t)n_pad * sizeof(T), s));
  }
  CK(cudaEventRecord(ctx->ev[2], s));

  // ---- Cholesky (forward substitution of delta rides along in the border tile)
  cholesky_inplace<T>(ctx, L, lda, n_pad, lda, Dinv, dscal, dinfo);
  CK(cudaEventRecord(ctx->ev[3], s));

  // ---- sqmahal, alpha = L^-T v, logpdf
  if (S > 0) {
    launch_extract_v<T>(L, lda, n_pad, S, rwork, dscal + nblk, s);
    if (alpha_out || keep) {
      launch_bwd_solve<T>(L, lda, Dinv, nblk, rwork, dflags, s);
      CK(cudaMemcpyAsync(alpha, rwork, (size_t)n_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
    }
  }
  launch_finalize_logpdf<T>(dscal, nblk, dscal + nblk, S, N, lp_d, dscal + nblk + TILE, s);
  CK(cudaEventRecord(ctx->ev[4], s));

  // ---- D2H
  int h_info = 0;
  double h_logdet = 0.0;
  CK(cudaMemcpyAsync(&h_info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&h_logdet, dscal + nblk + TILE, sizeof(double), cudaMemcpyDeviceToHost, s));
  if (S > 0 && logpdf_out) CK(cudaMemcpyAsync(logpdf_out, lp_d, (size_t)S * sizeof(T), cudaMemcpyDeviceToHost, s));
  if (S > 0 && alpha_out) { rc = download<T>(ctx, alpha_out, alpha, (size_t)N, false); if (rc) return rc; }
  CK(cudaEventRecord(ctx->ev[5], s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());

  float ms = 0;
  auto el = [&](int a, int b) { cudaEventElapsedTime(&ms, ctx->ev[a], ctx->ev[b]); return (double)ms; };
  ctx->timings[0] = el(0, 5); ctx->timings[1] = el(0, 1); ctx->timings[2] = el(1, 2); ctx->timings[3] = el(2, 3);
  ctx->timings[4] = el(3, 4); ctx->timings[5] = el(4, 5); ctx->timings[6] = 0.0;
  ctx->timings[7] = ctx->profile ? prof_total_ms(ctx) : 0.0;

  if (h_info != 0) {
    ctx->info = h_info;
    char b[128];
    snprintf(b, sizeof(b), "matrix is not positive definite; Cholesky failed at pivot %d", h_info);
    ctx->err = b;
    return AGP_ERR_NOT_POSDEF;  // the guard releases the handle
  }
  pguard.p = nullptr;
  if (post) { post->logdet = h_logdet; *post_out = post; }
  if (L_keep) { *L_keep = L; *lda_out = lda; }
  return AGP_OK;
}

// logpdf(fx, Y::Matrix) has no limit on the number of columns (/root/reference/src/finite_gp_projection.jl:306-311).
// The border tile carries 128 right-hand sides through the factorisation; further columns reuse the SAME factor:
// V = L^-1 (Y_c - m) by the multi-RHS forward substitution, sqmahal = column sums of V.^2 -- ONE Gram and ONE Cholesky
// whatever S is.
template <typename T>
int fit_many_impl(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout,
                  const void* X, int64_t N, int D, const void* Y, int S, void* logpdf_out, void* alpha_out,
                  agp_post** post_out) {
  if (S <= TILE) return fit_impl<T>(ctx, k, mean, noise, layout, X, N, D, Y, S, logpdf_out, alpha_out, post_out, nullptr, nullptr, nullptr);
  if (!Y || !logpdf_out) { ctx->err = "Y/logpdf_out is NULL"; return AGP_ERR_INVALID; }
  agp_post* p = nullptr;
  int rc = fit_impl<T>(ctx, k, mean, noise, layout, X, N, D, Y, TILE, logpdf_out, alpha_out, &p, nullptr, nullptr, nullptr);
  if (rc) return rc;
  struct Guard { agp_post* p; bool keep; ~Guard() { if (p && !keep) agp_post_free(p); } } guard{p, false};
  cudaStream_t s = ctx->stream;
  static const agp_mean zero_mean{0, 0.0, nullptr};
  if (!mean) mean = &zero_mean;
  const int64_t n_pad = p->n_pad;
  const double log2pi = 1.8378770664093454835606594728112;
  const int64_t chunk = 1024;
  Scratch sc(ctx);
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)n_pad * chunk * sizeof(T)));
  T* B = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)chunk * sizeof(T)));
  T* sq = (T*)tmp;
  T* mean_d = nullptr;
  if (mean->kind == 2) { rc = upload<T>(ctx, sc, mean->v, N, true, &mean_d); if (rc) return rc; }
  std::vector<T> h_sq((size_t)chunk);
  for (int64_t c0 = TILE; c0 < S; c0 += chunk) {
    const int64_t nc = (S - c0 < chunk) ? (S - c0) : chunk, nc_pad = round_up(nc, TILE);
    Scratch scc(ctx);
    T* Yd = nullptr;
    rc = upload<T>(ctx, scc, (const T*)Y + (size_t)c0 * N, (size_t)N * nc, false, &Yd);
    if (rc) return rc;
    CK(cudaMemsetAsync(B, 0, (size_t)n_pad * nc_pad * sizeof(T), s));
    CK(cudaMemsetAsync(sq, 0, (size_t)chunk * sizeof(T), s));
    for (int64_t j = 0; j < nc; ++j) launch_sub_mean<T>(Yd + j * N, N, mean->kind, mean->c, mean_d, B + j * n_pad, s);
    forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, B, n_pad, nc_pad);
    launch_colsumsq_acc<T>(B, n_pad, n_pad, nc, 1.0, sq, s);
    CK(cudaMemcpyAsync(h_sq.data(), sq, (size_t)nc * sizeof(T), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (int64_t j = 0; j < nc; ++j)
      ((T*)logpdf_out)[c0 + j] = (T)(-0.5 * ((double)N * log2pi + p->logdet + (double)h_sq[(size_t)j]));
  }
  CK(cudaGetLastError());
  if (post_out) { *post_out = p; guard.keep = true; }
  return AGP_OK;
}

// rows [c0, c0 + mc) of a feature-major point set (M x D column-major, host or device per the context's memspace) gathered
// into a contiguous mc x D feature-major DEVICE block: chunked prediction over RowVecs inputs larger than one chunk
template <typename T>
int gather_feature_major_chunk(agp_ctx* ctx, Scratch& sc, const void* Xs, int64_t M, int D, int64_t c0, int64_t mc, T** out) {
  void* d = nullptr;
  CK(sc.alloc(&d, (size_t)mc * D * sizeof(T)));
  const cudaMemcpyKind kind = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  CK(cudaMemcpy2DAsync(d, (size_t)mc * sizeof(T), (const T*)Xs + c0, (size_t)M * sizeof(T), (size_t)mc * sizeof(T), (size_t)D, kind,
                       ctx->stream));
  *out = (T*)d;
  return AGP_OK;
}

template <typename T>
int post_cross(agp_post* p, Scratch& sc, int layout, const void* Xs, int64_t M, int64_t m_pad, T** Xst, T** B) {
  agp_ctx* ctx = p->ctx;
  int rc = prep_points<T>(ctx, sc, &p->k, (const T*)p->ard, layout, Xs, M, m_pad, p->D, Xst, false);
  if (rc) return rc;
  void* b = nullptr;
  CK(sc.alloc(&b, (size_t)p->n_pad * m_pad * sizeof(T)));
  *B = (T*)b;
  GramParams gp{};
  fill_gram_params<T>(gp, &p->k, 0, 0, p->n, M, nullptr, nullptr, p->comp);
  gp.mask_a = p->valid;
  launch_gram<T>((const T*)p->Xt, *Xst, p->n_pad, m_pad, p->D, *B, p->n_pad, gp, ctx->stream);
  return AGP_OK;
}

template <typename T>
int post_mean_var_impl(agp_post* p, int layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                       const agp_noise* noise_s, void* mean_out, void* var_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (M <= 0) return AGP_OK;
  CK(cudaEventRecord(ctx->ev[0], s));
  // chunk the test points so that the N x Mc cross-Gram stays <= ~4 GB
  int64_t cap = (int64_t)(4.0e9 / ((double)p->n_pad * sizeof(T)));
  { const int64_t c_env = env_int64("AGP_PREDICT_CHUNK", 0); if (c_env > 0) cap = c_env; }  // tests: force small chunks
  cap = cap / TILE * TILE;
  if (cap < TILE) cap = TILE;
  agp_mean mz{p->mean_kind, p->mean_c, nullptr};
  if (!mean_s) mean_s = &mz;
  for (int64_t c0 = 0; c0 < M; c0 += cap) {
    const int64_t mc = (M - c0 < cap) ? (M - c0) : cap;
    const int64_t m_pad = round_up(mc, TILE);
    Scratch sc(ctx);
    const char* xs_c = (const char*)Xs;
    const void* xs_chunk = nullptr;
    const int saved_memspace = ctx->memspace;
    if (layout == AGP_POINT_MAJOR) {
      xs_chunk = xs_c + (size_t)c0 * p->D * sizeof(T);
    } else if (c0 == 0 && mc == M) {
      xs_chunk = Xs;
    } else {  // RowVecs test set larger than one chunk: gather the chunk's rows on the device
      T* g = nullptr;
      int grc = gather_feature_major_chunk<T>(ctx, sc, Xs, M, p->D, c0, mc, &g);
      if (grc) return grc;
      xs_chunk = g;
      ctx->memspace = AGP_MEM_DEVICE;  // the gathered block is a device pointer (inputs only; outputs use the override below)
    }
    T *Xst = nullptr, *B = nullptr;
    int rc = post_cross<T>(p, sc, layout, xs_chunk, mc, m_pad, &Xst, &B);
    const bool out_dev_saved = ctx->out_dev_override;
    if (ctx->memspace != saved_memspace) { ctx->memspace = saved_memspace; }
    (void)out_dev_saved;
    if (rc) return rc;
    T *mean_d = nullptr, *noise_d = nullptr;
    if (mean_s->kind == 2) { rc = upload<T>(ctx, sc, (const T*)mean_s->v + c0, mc, true, &mean_d); if (rc) return rc; }
    if (noise_s && noise_s->kind == 1) { rc = upload<T>(ctx, sc, (const T*)noise_s->v + c0, mc, true, &noise_d); if (rc) return rc; }
    void* tmp = nullptr;
    CK(sc.alloc(&tmp, (size_t)m_pad * 3 * sizeof(T)));
    T* mu = (T*)tmp; T* var = mu + m_pad; T* kd = var + m_pad;
    launch_kdiag<T>(Xst, mc, p->D, p->k.family, p->k.variance, p->k.linear_c, kd, s, p->comp ? &p->comp->desc : nullptr);
    launch_gemv_t<T>(B, p->n_pad, p->n_pad, mc, (const T*)p->alpha, mean_s->kind, mean_s->c, mean_d, mu, s);
    if (var_out) {
      forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, p->n_pad, B, p->n_pad, m_pad);
      launch_colsumsq_var<T>(B, p->n_pad, p->n_pad, mc, kd, noise_s ? noise_s->kind : -1, noise_s ? noise_s->s : 0.0,
                             noise_d, var, s);
    }
    if (mean_out) { rc = download<T>(ctx, (T*)mean_out + c0, mu, mc, false); if (rc) return rc; }
    if (var_out) { rc = download<T>(ctx, (T*)var_out + c0, var, mc, false); if (rc) return rc; }
    CK(cudaStreamSynchronize(s));
  }
  CK(cudaEventRecord(ctx->ev[1], s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]);
  ctx->timings[6] = ms;
  ctx->timings[0] = ms;
  return AGP_OK;
}


// ---- distributed posterior: gather the block-column-cyclic factor so that every rank holds it whole (SURVEY s8e:
// "partition the M test points across GPUs if the factor is replicated").  Collective: every rank of the communicator
// calls it at the same point (all handle operations are SPMD, like agp_fit on a distributed context).
template <typename T>
int post_replicate(agp_post* p) {
  if (!p->Lloc) return AGP_OK;
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  const int R = p->dist_R, me = p->dist_me, G = p->dist_G;
  const int64_t W = p->dist_W, lda = p->lda, n_pad = p->n_pad;
  const int nto = (int)(n_pad / W), nt = (int)(n_pad / TILE);
  void *Lf = nullptr, *Df = nullptr;
  CK(cudaMallocAsync(&Lf, (size_t)lda * n_pad * sizeof(T), s));
  CK(cudaMallocAsync(&Df, (size_t)nt * TILE * TILE * sizeof(T), s));
  for (int jo = 0; jo < nto; ++jo) {
    const int owner = jo % R, lj = jo / R;
    T* dstL = (T*)Lf + (int64_t)jo * W * lda;
    T* dstD = (T*)Df + (int64_t)jo * G * TILE * TILE;
    const T* srcL = owner == me ? (const T*)p->Lloc + (int64_t)lj * W * lda : dstL;
    const T* srcD = owner == me ? (const T*)p->Dinv_loc + (int64_t)lj * G * TILE * TILE : dstD;
    CKN(ncclBroadcast(srcL, dstL, (size_t)lda * W, NcclType<T>::v, owner, ctx->nccl, s));
    CKN(ncclBroadcast(srcD, dstD, (size_t)G * TILE * TILE, NcclType<T>::v, owner, ctx->nccl, s));
  }
  CK(cudaStreamSynchronize(s));
  cudaFreeAsync(p->Lloc, s);
  cudaFreeAsync(p->Dinv_loc, s);
  p->Lloc = nullptr; p->Dinv_loc = nullptr;
  p->L = Lf; p->Dinv = Df;
  return AGP_OK;
}

// mean_and_var over a distributed posterior: the factor is replicated (once), the test points are partitioned over the
// ranks (point-major inputs), every rank predicts its slice with the single-GPU path and the M-vectors are exchanged
// with one broadcast per rank.  Every rank returns the complete outputs.
template <typename T>
int post_mean_var_dist(agp_post* p, int layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                       const agp_noise* noise_s, void* mean_out, void* var_out) {
  agp_ctx* ctx = p->ctx;
  int rc = post_replicate<T>(p);
  if (rc) return rc;
  const int R = p->dist_R, me = p->dist_me;
  if (layout != AGP_POINT_MAJOR || M < 2 * R)  // small or feature-major: every rank computes everything (same result)
    return post_mean_var_impl<T>(p, layout, Xs, M, mean_s, noise_s, mean_out, var_out);
  cudaStream_t s = ctx->stream;
  Scratch sc(ctx);
  const int64_t per = (M + R - 1) / R, lo = (int64_t)me * per < M ? (int64_t)me * per : M;
  const int64_t hi = lo + per < M ? lo + per : M;
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)2 * M * sizeof(T)));
  T* mu_all = (T*)tmp; T* var_all = mu_all + M;
  agp_mean ms; agp_noise ns;
  const agp_mean* msp = nullptr; const agp_noise* nsp = nullptr;
  if (mean_s) { ms = *mean_s; if (ms.kind == 2 && ms.v) ms.v = (const T*)ms.v + lo; msp = &ms; }
  if (noise_s) { ns = *noise_s; if (ns.kind == 1 && ns.v) ns.v = (const T*)ns.v + lo; nsp = &ns; }
  if (hi > lo) {
    ctx->out_dev_override = true;
    rc = post_mean_var_impl<T>(p, layout, (const char*)Xs + (size_t)lo * p->D * sizeof(T), hi - lo, msp, nsp,
                               mean_out ? mu_all + lo : nullptr, var_out ? var_all + lo : nullptr);
    ctx->out_dev_override = false;
    if (rc) return rc;
  }
  for (int r = 0; r < R; ++r) {
    const int64_t rlo = (int64_t)r * per < M ? (int64_t)r * per : M, rhi = rlo + per < M ? rlo + per : M;
    if (rhi <= rlo) continue;
    if (mean_out) CKN(ncclBroadcast(mu_all + rlo, mu_all + rlo, (size_t)(rhi - rlo), NcclType<T>::v, r, ctx->nccl, s));
    if (var_out) CKN(ncclBroadcast(var_all + rlo, var_all + rlo, (size_t)(rhi - rlo), NcclType<T>::v, r, ctx->nccl, s));
  }
  if (mean_out) { rc = download<T>(ctx, mean_out, mu_all, (size_t)M, false); if (rc) return rc; }
  if (var_out) { rc = download<T>(ctx, var_out, var_all, (size_t)M, false); if (rc) return rc; }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

template <typename T>
int post_mean_cov_impl(agp_post* p, int layout, const void* Xs, int64_t M, const agp_mean* mean_s, void* mean_out,
                       void* cov_out) {
  agp_ctx* ctx = p->ctx;
  { int rrc = post_replicate<T>(p); if (rrc) return rrc; }
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (M <= 0) return AGP_OK;
  const int64_t m_pad = round_up(M, TILE);
  Scratch sc(ctx);
  T *Xst = nullptr, *B = nullptr;
  int rc = post_cross<T>(p, sc, layout, Xs, M, m_pad, &Xst, &B);
  if (rc) return rc;
  agp_mean mz{p->mean_kind, p->mean_c, nullptr};
  if (!mean_s) mean_s = &mz;
  T* mean_d = nullptr;
  if (mean_s->kind == 2) { rc = upload<T>(ctx, sc, mean_s->v, M, true, &mean_d); if (rc) return rc; }
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)m_pad * sizeof(T)));
  T* mu = (T*)tmp;
  launch_gemv_t<T>(B, p->n_pad, p->n_pad, M, (const T*)p->alpha, mean_s->kind, mean_s->c, mean_d, mu, s);
  if (mean_out) { rc = download<T>(ctx, mean_out, mu, M, false); if (rc) return rc; }
  if (cov_out) {
    forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, p->n_pad, B, p->n_pad, m_pad);
    CK(sc.alloc(&tmp, (size_t)m_pad * m_pad * sizeof(T) * 2));
    T* C = (T*)tmp; T* Kss = C + m_pad * m_pad;
    GemmArgs g{};  // C = V' V
    g.A = B; g.lda = p->n_pad; g.a_kmajor = 1;
    g.B = B; g.ldb = p->n_pad; g.b_kmajor = 1;
    g.C = C; g.ldc = m_pad; g.M = m_pad; g.N = m_pad; g.K = p->n_pad;
    launch_gemm<T>(g, s);
    GramParams gp{};
    fill_gram_params<T>(gp, &p->k, 1, 0, M, M, nullptr, nullptr, p->comp);
    launch_gram<T>(Xst, Xst, m_pad, m_pad, p->D, Kss, m_pad, gp, s);
    launch_cov_finish<T>(C, m_pad, Kss, m_pad, s);
    cudaMemcpyKind kind = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    CK(cudaMemcpy2DAsync(cov_out, (size_t)M * sizeof(T), C, (size_t)m_pad * sizeof(T), (size_t)M * sizeof(T), (size_t)M, kind, s));
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// ---- logpdf / rand of a FiniteGP over a posterior: logpdf(f_post(x*, Sigma*), Y) and rand(f_post(x*, Sigma*), S)
// (/root/reference/src/finite_gp_projection.jl:306-311 and :233-237 applied to f = PosteriorGP, whose
// mean_and_cov is /root/reference/src/exact_gpr_posterior.jl:78-83).  The M x M posterior covariance never
// leaves the device: K** + Sigma* is generated straight into a factor buffer, V'V (V = L^-1 K(x, x*)) is
// subtracted by one GEMM, and the same in-place Cholesky as agp_fit runs with (Y - m*)' in the border tile.

// the test-side defaults of agp_post_logpdf / agp_post_rand / agp_post_pred_logpdf_grad: the handle's mean, and
// default_sigma^2 (finite_gp_projection.jl:17) for the noise.  handle_mean holds the default mean for the call.
inline int post_side_defaults(agp_post* p, const agp_mean** mean_s, const agp_noise** noise_s, agp_mean* handle_mean) {
  agp_ctx* ctx = p->ctx;
  static const agp_noise default_noise{0, 1e-18, nullptr};
  if (!*noise_s) *noise_s = &default_noise;
  if ((*noise_s)->kind == 1 && !(*noise_s)->v) { ctx->err = "noise vector is NULL"; return AGP_ERR_INVALID; }
  *handle_mean = agp_mean{p->mean_kind, p->mean_c, nullptr};
  if (!*mean_s) *mean_s = handle_mean;
  if ((*mean_s)->kind == 2 && !(*mean_s)->v) { ctx->err = "mean vector is NULL"; return AGP_ERR_INVALID; }
  return AGP_OK;
}

// C* + Sigma* = K(x*, x*) + Sigma* - A'A (A = L^-1 K(x, x*), the handle's n_pad rows), lower triangle, with (Y - mu)' in
// the border (S columns; none with S = 0), factored in place by agp_fit's Cholesky.  Into the call's scratch: Lf_out the
// factor (leading dimension m_pad + TILE, identity padding), Dinv_out its inverted diagonal blocks, dscal_out the
// per-block log-determinants (then the border's sums), dinfo_out the failed pivot (read by post_cov_status).
template <typename T>
int post_cov_factor(agp_post* p, Scratch& sc, const T* Xst, const T* A, int64_t M, const agp_noise* noise_s,
                    const T* noise_d, const T* Yd, int S, const T* mu, T** Lf_out, T** Dinv_out, double** dscal_out,
                    int** dinfo_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  const int64_t m_pad = round_up(M, TILE), ldf = m_pad + TILE;
  const int nblk = (int)(m_pad / TILE);
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)ldf * m_pad * sizeof(T)));
  T* Lf = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)nblk * TILE * TILE * sizeof(T)));
  T* Dinv = (T*)tmp;
  GramParams gp{};
  fill_gram_params<T>(gp, &p->k, 1, 1, M, M, noise_s, noise_d, p->comp);
  launch_gram<T>(Xst, Xst, m_pad, m_pad, p->D, Lf, ldf, gp, s);
  {
    GemmArgs g{};
    g.A = A; g.lda = p->n_pad; g.a_kmajor = 1;
    g.B = A; g.ldb = p->n_pad; g.b_kmajor = 1;
    g.C = Lf; g.ldc = ldf; g.M = m_pad; g.N = m_pad; g.K = p->n_pad;
    g.alpha_neg = 1; g.beta_one = 1; g.lower_only = 1;
    launch_gemm<T>(g, s);
  }
  launch_border_init<T>(Lf, ldf, M, m_pad, Yd, M, S, 2, 0.0, mu, s);  // border = (Y - mu)'
  CK(sc.alloc(&tmp, (size_t)(nblk + TILE + 2) * sizeof(double)));
  double* dscal = (double*)tmp;
  CK(sc.alloc(&tmp, sizeof(int)));
  int* dinfo = (int*)tmp;
  CK(cudaMemsetAsync(dinfo, 0, sizeof(int), s));
  prof_begin(ctx);
  cholesky_inplace<T>(ctx, Lf, ldf, m_pad, ldf, Dinv, dscal, dinfo);
  *Lf_out = Lf; *Dinv_out = Dinv; *dscal_out = dscal; *dinfo_out = dinfo;
  return AGP_OK;
}

// waits for the stream and reports a failed factorisation of the posterior covariance
inline int post_cov_status(agp_ctx* ctx, const int* dinfo) {
  int h_info = 0;
  CK(cudaMemcpyAsync(&h_info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaGetLastError());
  if (h_info != 0) {
    ctx->info = h_info;
    char b[128];
    snprintf(b, sizeof(b), "posterior covariance is not positive definite; Cholesky failed at pivot %d", h_info);
    ctx->err = b;
    return AGP_ERR_NOT_POSDEF;
  }
  return AGP_OK;
}

template <typename T>
int post_cond_impl(agp_post* p, int layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                   const agp_noise* noise_s, const void* Y, int S, void* logpdf_out, const void* Z, int Sz,
                   void* rand_out) {
  agp_ctx* ctx = p->ctx;
  { int rrc = post_replicate<T>(p); if (rrc) return rrc; }
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (M <= 0) { ctx->err = "M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (!Xs) { ctx->err = "Xs is NULL"; return AGP_ERR_INVALID; }
  if (S < 0 || S > TILE) { ctx->err = "number of right-hand sides must be in [0,128]"; return AGP_ERR_UNSUPPORTED; }
  if (S > 0 && (!Y || !logpdf_out)) { ctx->err = "Y/logpdf_out is NULL"; return AGP_ERR_INVALID; }
  if (Sz > 0 && (!Z || !rand_out)) { ctx->err = "Z/out is NULL"; return AGP_ERR_INVALID; }
  agp_mean mz;
  int rc = post_side_defaults(p, &mean_s, &noise_s, &mz);
  if (rc) return rc;

  const int64_t m_pad = round_up(M, TILE), ldf = m_pad + TILE;
  const int nblk = (int)(m_pad / TILE);
  Scratch sc(ctx);
  T *Xst = nullptr, *B = nullptr;
  rc = post_cross<T>(p, sc, layout, Xs, M, m_pad, &Xst, &B);
  if (rc) return rc;
  T *mean_d = nullptr, *noise_d = nullptr, *Yd = nullptr;
  if (mean_s->kind == 2) { rc = upload<T>(ctx, sc, mean_s->v, M, true, &mean_d); if (rc) return rc; }
  if (noise_s->kind == 1) { rc = upload<T>(ctx, sc, noise_s->v, M, true, &noise_d); if (rc) return rc; }
  if (S > 0) { rc = upload<T>(ctx, sc, Y, (size_t)M * S, false, &Yd); if (rc) return rc; }
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)m_pad * sizeof(T)));
  T* mu = (T*)tmp;
  CK(cudaMemsetAsync(mu, 0, (size_t)m_pad * sizeof(T), s));
  // posterior mean m* = m(x*) + K(x*, x) alpha, then V = L^-1 K(x, x*) in place
  launch_gemv_t<T>(B, p->n_pad, p->n_pad, M, (const T*)p->alpha, mean_s->kind, mean_s->c, mean_d, mu, s);
  forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, p->n_pad, B, p->n_pad, m_pad);
  T *Lf = nullptr, *Dinv = nullptr;
  double* dscal = nullptr;
  int* dinfo = nullptr;
  rc = post_cov_factor<T>(p, sc, Xst, B, M, noise_s, noise_d, Yd, S, mu, &Lf, &Dinv, &dscal, &dinfo);
  if (rc) return rc;
  CK(sc.alloc(&tmp, (size_t)TILE * sizeof(T)));
  T* lp_d = (T*)tmp;
  if (S > 0) {
    CK(sc.alloc(&tmp, (size_t)S * m_pad * sizeof(T)));
    launch_extract_v<T>(Lf, ldf, m_pad, S, (T*)tmp, dscal + nblk, s);
    launch_finalize_logpdf<T>(dscal, nblk, dscal + nblk, S, M, lp_d, dscal + nblk + TILE, s);
  }
  rc = post_cov_status(ctx, dinfo);
  if (rc) return rc;
  if (S > 0) CK(cudaMemcpyAsync(logpdf_out, lp_d, (size_t)S * sizeof(T), cudaMemcpyDeviceToHost, s));
  if (Sz > 0) {  // out = m* + L* Z  (C.U' * randn, finite_gp_projection.jl:235)
    const int64_t s_pad = round_up(Sz, 4);
    CK(sc.alloc(&tmp, (size_t)m_pad * s_pad * sizeof(T) * 2));
    T* Zd = (T*)tmp; T* Od = Zd + m_pad * s_pad;
    CK(cudaMemsetAsync(Zd, 0, (size_t)m_pad * s_pad * sizeof(T), s));
    cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    CK(cudaMemcpy2DAsync(Zd, (size_t)m_pad * sizeof(T), Z, (size_t)M * sizeof(T), (size_t)M * sizeof(T), (size_t)Sz, kin, s));
    GemmArgs g{};
    g.A = Lf; g.lda = ldf; g.a_kmajor = 0;
    g.B = Zd; g.ldb = m_pad; g.b_kmajor = 1;
    g.C = Od; g.ldc = m_pad; g.M = m_pad; g.N = s_pad; g.K = m_pad; g.trmm_lower = 1;
    launch_gemm<T>(g, s);
    launch_add_mean_cols<T>(Od, m_pad, M, Sz, 2, 0.0, (const T*)mu, s);
    CK(cudaMemcpy2DAsync(rand_out, (size_t)M * sizeof(T), Od, (size_t)m_pad * sizeof(T), (size_t)M * sizeof(T), (size_t)Sz, kout, s));
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// ---- EXPERIMENTAL (compiles, not yet run on a device): gradient of logpdf(fx, y) w.r.t. the hyper-parameters from the
// factor agp_fit left in the handle (SURVEY s8f rank 1).  V = L^-1 by the blocked forward
// substitution on the identity, C^-1 = V'V by the lower-only GEMM (both validated kernels), then grad.cu's fused
// reduction 1/2 sum (alpha alpha' - C^-1) o dC/dtheta.  Extra cost ~ 2 N^3 flop and two N^2 buffers.
// a single kernel as a one-factor descriptor over its transformed points (grad_x.cu); its Scale / ARD chain factor is
// applied by the caller
static CompositeDesc single_kernel_desc(int family, double variance, double linear_c) {
  CompositeDesc one{};
  one.nterms = 1; one.nfactors = 1; one.nacc = 1;
  one.variance[0] = variance;
  one.f[0].family = family; one.f[0].transform = AGP_T_NONE; one.f[0].acc = 0; one.f[0].term = 0;
  one.f[0].s = 1.0; one.f[0].s2 = 1.0; one.f[0].param = linear_c;
  one.f[0].g_s = one.f[0].g_p = one.f[0].g_w = one.f[0].g_r = -1;
  one.acc_kind[0] = family == AGP_LINEAR ? COMP_ACC_DOT : COMP_ACC_SQ;
  one.w = nullptr;
  return one;
}

// the single-kernel slots of a gradient (agp.h's layout) from grad_reduce_kernel's sums h: [0] variance, [1] the Scale
// factor, [2] LinearKernel c and [5..] the ARD values (ard_h, host copy of the transform's); slots 3 and 4 are the
// caller's
template <typename T>
void single_kernel_grad(const agp_kernel& k, int D, const double* h, const T* ard_h, double* grad_out) {
  const bool linear = k.family == AGP_LINEAR;
  const bool want_ard = k.transform == AGP_T_ARD;
  const double var = k.variance, sc_ = k.scale;
  grad_out[0] = 0.5 * h[0];
  grad_out[1] = (k.transform == AGP_T_SCALE) ? (linear ? var * h[1] / sc_ : 0.5 * var * h[1] / sc_) : 0.0;
  grad_out[2] = linear ? 0.5 * var * h[2] : 0.0;
  for (int d = 0; d < D; ++d)
    grad_out[5 + d] = want_ard ? (linear ? var : 0.5 * var) * h[(size_t)5 + d] / (double)ard_h[(size_t)d] : 0.0;
}

// sum_i v_i of a device vector on the host, in index order and in double
template <typename T>
int host_sum(agp_ctx* ctx, const T* v, int64_t n, double* out) {
  std::vector<T> h((size_t)n);
  CK(cudaMemcpyAsync(h.data(), v, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  double c = 0.0;
  for (int64_t i = 0; i < n; ++i) c += (double)h[(size_t)i];
  *out = c;
  return AGP_OK;
}

// The reductions that end every gradient of this form, on the handle's points and kernel: with W = alpha alpha' - Cinv
// (Cinv: its lower tiles are read, leading dimension n_pad),
//   grad_out = the agp_post_logpdf_grad layout of 1/2 sum_ij W_ij dC_ij/dtheta ([3] = 1/2 tr W, [4] = sum alpha),
//   noise_diag_out = 1/2 W_ii,  x_grad_out = sum_j W_ij d1k(x_i, x_j)  (agp_post_logpdf_grad_x).
// Any output may be NULL.  agp_post_logpdf_grad_x runs it with C^-1; agp_rand_grad with alpha = 0 and Cinv = -V'QV.
// grad_reductions_on runs the same reductions with the handle's kernel over another point set X (n points, n_pad rows,
// transformed like the handle's) and a W of leading dimension ldc: agp_post_pred_logpdf_grad's stacked [x; x*].
template <typename T>
int grad_reductions_on(agp_post* p, Scratch& sc, const T* X, int64_t n, int64_t n_pad, const T* Cinv, int64_t ldc,
                       const T* alpha, double* grad_out, void* noise_diag_out, int layout, void* x_grad_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  const int D = p->D;
  const bool want_theta = grad_out || noise_diag_out;  // the hyper-parameter reduction also yields noise_diag
  void* tmp = nullptr;
  const int64_t nsums = agp_post_grad_len(p);  // 5 + D for a single kernel
  CK(sc.alloc(&tmp, (size_t)nsums * sizeof(double)));
  double* sums = (double*)tmp;
  T* noise_d = nullptr;
  if (noise_diag_out) { CK(sc.alloc(&tmp, (size_t)n_pad * sizeof(T))); noise_d = (T*)tmp; }
  CK(cudaMemsetAsync(sums, 0, (size_t)nsums * sizeof(double), s));
  const int want_ard = (p->k.transform == AGP_T_ARD) ? 1 : 0;
  if (want_theta) {
    if (p->comp)
      launch_composite_grad_reduce<T>(X, D, n, n_pad, Cinv, ldc, alpha, p->comp->desc, sums, noise_d, s);
    else
      launch_grad_reduce<T>(X, D, n, n_pad, Cinv, ldc, alpha, p->k.family, p->k.linear_c, want_ard, sums, noise_d, s);
  }
  if (x_grad_out) {  // sum_j W_ij d1k(x_i, x_j) from the same W (grad_x.cu)
    const CompositeDesc one = single_kernel_desc(p->k.family, p->k.variance, p->k.linear_c);
    const CompositeDesc* cd = &one;
    double mult = 1.0;
    const T* ard = nullptr;
    if (p->comp) {
      cd = &p->comp->desc;
    } else {
      if (p->k.transform == AGP_T_SCALE) mult = p->k.scale;
      else if (want_ard) ard = (const T*)p->ard;
    }
    CK(sc.alloc(&tmp, (size_t)grad_x_part_len(n, D, cd->nacc) * sizeof(double)));
    double* part = (double*)tmp;
    CK(sc.alloc(&tmp, (size_t)n * D * sizeof(T)));
    T* xg = (T*)tmp;
    launch_grad_x<T>(X, D, n, Cinv, ldc, alpha, *cd, mult, ard, layout, part, xg, s);
    int rc = download<T>(ctx, x_grad_out, xg, (size_t)n * D, false); if (rc) return rc;
  }
  if (!want_theta) {
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    return AGP_OK;
  }
  if (p->comp) {  // composite: every kernel slot is 1/2 sum_ij W_ij dK_ij/dtheta, already in its final place
    std::vector<double> h((size_t)nsums);
    CK(cudaMemcpyAsync(h.data(), sums, h.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (noise_diag_out) { int rc = download<T>(ctx, noise_diag_out, noise_d, (size_t)n, false); if (rc) return rc; }
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    if (!grad_out) return AGP_OK;
    for (int64_t i = 0; i < nsums; ++i) grad_out[i] = 0.5 * h[(size_t)i];
    grad_out[0] = grad_out[1] = grad_out[2] = 0.0;
    grad_out[4] = h[4];
    return AGP_OK;
  }
  std::vector<double> h((size_t)5 + D);
  std::vector<T> ard_h((size_t)(D > 0 ? D : 1));
  CK(cudaMemcpyAsync(h.data(), sums, h.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (want_ard && p->ard) CK(cudaMemcpyAsync(ard_h.data(), p->ard, (size_t)D * sizeof(T), cudaMemcpyDeviceToHost, s));
  if (noise_diag_out) { int rc = download<T>(ctx, noise_diag_out, noise_d, (size_t)n, false); if (rc) return rc; }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (!grad_out) return AGP_OK;
  single_kernel_grad<T>(p->k, D, h.data(), ard_h.data(), grad_out);
  grad_out[3] = 0.5 * h[3];
  grad_out[4] = h[4];
  return AGP_OK;
}

template <typename T>
int grad_reductions(agp_post* p, Scratch& sc, const T* Cinv, const T* alpha, double* grad_out, void* noise_diag_out, int layout,
                    void* x_grad_out) {
  return grad_reductions_on<T>(p, sc, (const T*)p->Xt, p->n, p->n_pad, Cinv, p->n_pad, alpha, grad_out, noise_diag_out,
                               layout, x_grad_out);
}


inline int check_layout(agp_ctx* ctx, int layout) {
  if (layout != AGP_POINT_MAJOR && layout != AGP_FEATURE_MAJOR) { ctx->err = "layout must be AGP_POINT_MAJOR or AGP_FEATURE_MAJOR"; return AGP_ERR_INVALID; }
  return AGP_OK;
}

// what every logpdf gradient of a handle checks first: the input layout, the factor gathered whole, a handle straight
// from agp_fit
template <typename T>
int logpdf_grad_prelude(agp_post* p, int layout) {
  agp_ctx* ctx = p->ctx;
  { int rc = check_layout(ctx, layout); if (rc) return rc; }
  { int rrc = post_replicate<T>(p); if (rrc) return rrc; }
  CK(cudaSetDevice(ctx->device));
  if (p->valid || p->segs.size() > 1) { ctx->err = "gradient of an extended (sequentially conditioned) posterior is unsupported"; return AGP_ERR_UNSUPPORTED; }
  return AGP_OK;
}

// V = L^-1 by the blocked forward substitution on the identity and, with want_cinv, C^-1 = V'V into its lower tiles: two
// n_pad x n_pad buffers of the call's scratch (Cinv stays null without want_cinv)
template <typename T>
int inverse_factor(agp_post* p, Scratch& sc, bool want_cinv, T** V_out, T** Cinv_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  const int64_t n_pad = p->n_pad;
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)n_pad * n_pad * sizeof(T)));
  T* V = (T*)tmp;
  T* Cinv = nullptr;
  if (want_cinv) { CK(sc.alloc(&tmp, (size_t)n_pad * n_pad * sizeof(T))); Cinv = (T*)tmp; }
  CK(cudaMemsetAsync(V, 0, (size_t)n_pad * n_pad * sizeof(T), s));
  launch_add_diag<T>(V, n_pad, n_pad, 1.0, s);
  forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, V, n_pad, n_pad);
  if (want_cinv) {
    GemmArgs g{};  // C^-1 = V'V, lower tiles
    g.A = V; g.lda = n_pad; g.a_kmajor = 1;
    g.B = V; g.ldb = n_pad; g.b_kmajor = 1;
    g.C = Cinv; g.ldc = n_pad; g.M = n_pad; g.N = n_pad; g.K = n_pad; g.lower_only = 1;
    launch_gemm<T>(g, s);
  }
  *V_out = V; *Cinv_out = Cinv;
  return AGP_OK;
}

template <typename T>
int post_logpdf_grad_impl(agp_post* p, double* grad_out, void* noise_diag_out, int layout, void* x_grad_out) {
  int rc = logpdf_grad_prelude<T>(p, layout);
  if (rc) return rc;
  if (!grad_out && !noise_diag_out && !x_grad_out) return AGP_OK;
  Scratch sc(p->ctx);
  T *V = nullptr, *Cinv = nullptr;
  rc = inverse_factor<T>(p, sc, true, &V, &Cinv);
  if (rc) return rc;
  return grad_reductions<T>(p, sc, Cinv, (const T*)p->alpha, grad_out, noise_diag_out, layout, x_grad_out);
}

// The column pullback of sum_s w_s logpdf(N(m, C), Y[:, s]) shared by the _cols and the held-out gradients.  C = L L' has
// n rows (n_pad padded); L, lda, Dinv are its blocked factor and V = L^-1 (leading dimension n_pad).  The S columns of Y
// (n x S, the caller's memory space) go through in chunks of up to 1024 with delta = Y - m (m: mean kind / c / device
// vector), B_c = L^-1 delta_c, A_c = V' B_c = C^-1 delta_c and w = lp_bar (all ones when NULL):
//   negW  = (sum w) C^-1 - sum_c A_c diag(w_c) A_c'   (negW holds C^-1 on entry; its lower tiles only with lower_only)
//   mbar += A_c w_c,  y_bar_out = -A diag(w) (n x S, the caller's memory space),  sq_s += |L^-1 delta_s|^2.
// Each output may be NULL.  w and the two n_pad x min(S, 1024) chunk buffers stay in sc.
template <typename T>
int weighted_cols_pullback(agp_ctx* ctx, Scratch& sc, const T* L, int64_t lda, const T* Dinv, int64_t n_pad, const T* V,
                           int64_t n, const void* Y, int mean_kind, double mean_c, const T* mean_d, int S,
                           const double* lp_bar, bool lower_only, T* negW, T* mbar, void* y_bar_out, T* sq) {
  cudaStream_t s = ctx->stream;
  std::vector<double> w((size_t)S, 1.0);
  if (lp_bar) w.assign(lp_bar, lp_bar + S);
  double wsum = 0.0;
  for (double v : w) wsum += v;
  std::vector<T> hw((size_t)2 * S);  // w, then -w
  for (int j = 0; j < S; ++j) { hw[(size_t)j] = (T)w[(size_t)j]; hw[(size_t)S + j] = (T)-w[(size_t)j]; }
  T* wd = nullptr;
  int rc = upload<T>(ctx, sc, hw.data(), hw.size(), true, &wd);
  if (rc) return rc;
  const int64_t chunk = 1024, cmax = round_up(S < chunk ? S : chunk, TILE);
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)n_pad * cmax * sizeof(T) * 2));
  T* B = (T*)tmp;  // delta_c, L^-1 delta_c, then Ybar_c
  T* A = B + n_pad * cmax;
  if (negW && wsum != 1.0) launch_scale<T>(negW, n_pad * n_pad, wsum, s);
  const cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  for (int64_t c0 = 0; c0 < S; c0 += chunk) {
    const int64_t nc = (S - c0 < chunk) ? (S - c0) : chunk, nc_pad = round_up(nc, TILE);
    Scratch scc(ctx);
    T* Yd = nullptr;
    rc = upload<T>(ctx, scc, (const T*)Y + (size_t)c0 * n, (size_t)n * nc, false, &Yd);
    if (rc) return rc;
    launch_sub_mean_cols<T>(Yd, n, n, nc, mean_kind, mean_c, mean_d, B, n_pad, n_pad, nc_pad, s);
    forward_subst_multi<T>(ctx, L, lda, Dinv, n_pad, B, n_pad, nc_pad);
    if (sq) launch_colsumsq_acc<T>(B, n_pad, n, nc, 1.0, sq + c0, s);
    {
      GemmArgs g{};  // A_c = V' B_c
      g.A = V; g.lda = n_pad; g.a_kmajor = 1;
      g.B = B; g.ldb = n_pad; g.b_kmajor = 1;
      g.C = A; g.ldc = n_pad; g.M = n_pad; g.N = nc_pad; g.K = n_pad;
      launch_gemm<T>(g, s);
    }
    if (mbar) launch_gemv_n_acc<T>(A, n_pad, n, nc, wd + c0, mbar, s);
    CK(cudaMemcpyAsync(B, A, (size_t)n_pad * nc_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
    launch_scale_cols<T>(B, n_pad, n_pad, nc, wd + S + c0, s);  // Ybar_c = A_c diag(-w_c)
    if (negW) {
      GemmArgs g{};  // negW += Ybar_c A_c'
      g.A = B; g.lda = n_pad; g.a_kmajor = 0;
      g.B = A; g.ldb = n_pad; g.b_kmajor = 0;
      g.C = negW; g.ldc = n_pad; g.M = n_pad; g.N = n_pad; g.K = nc_pad; g.beta_one = 1; g.lower_only = lower_only ? 1 : 0;
      launch_gemm<T>(g, s);
    }
    if (y_bar_out)
      CK(cudaMemcpy2DAsync((T*)y_bar_out + (size_t)c0 * n, (size_t)n * sizeof(T), B, (size_t)n_pad * sizeof(T), (size_t)n * sizeof(T),
                           (size_t)nc, kout, s));
  }
  return AGP_OK;
}

// ---- pullback of sum_s w_s logpdf(fx, Y[:, s]) on a handle from agp_fit (agp.h agp_post_logpdf_grad_cols).  With
// delta_s = Y[:, s] - m, A = C^-1 [delta_1 .. delta_S] and w = lp_bar:
//   -W = (sum_s w_s) C^-1 - A diag(w) A'   into the lower tiles of the C^-1 buffer,  mbar = A w,  Ybar = -A diag(w)
// and then the reductions of agp_post_logpdf_grad_x with alpha = 0 and C^-1 replaced by -W.  The columns go through
// weighted_cols_pullback in chunks of up to 1024 (fit_many_impl's), A_c = V' B_c on the tile GEMM (V = L^-1, as C^-1 =
// V'V is formed: the same accuracy class).  Two n_pad x n_pad and two n_pad x 1024 buffers of T whatever S is.
template <typename T>
int post_logpdf_grad_cols_impl(agp_post* p, const agp_mean* mean, const void* Y, int S, const double* lp_bar,
                               double* grad_out, void* noise_diag_out, void* mean_diag_out, int layout, void* x_grad_out,
                               void* y_bar_out) {
  agp_ctx* ctx = p->ctx;
  if (S < 1) { ctx->err = "S must be >= 1"; return AGP_ERR_INVALID; }
  if (!Y) { ctx->err = "Y is NULL"; return AGP_ERR_INVALID; }
  if (mean && mean->kind == 2 && !mean->v) { ctx->err = "mean vector is NULL"; return AGP_ERR_INVALID; }
  int rc = logpdf_grad_prelude<T>(p, layout);
  if (rc) return rc;
  const bool want_w = grad_out || noise_diag_out || x_grad_out;
  const bool want_mbar = grad_out || mean_diag_out;
  if (!want_w && !want_mbar && !y_bar_out) return AGP_OK;
  const agp_mean handle_mean{p->mean_kind, p->mean_c, nullptr};
  if (!mean) mean = &handle_mean;
  cudaStream_t s = ctx->stream;
  const int64_t N = p->n, n_pad = p->n_pad;
  Scratch sc(ctx);
  T *V = nullptr, *Cinv = nullptr;  // Cinv becomes -W
  rc = inverse_factor<T>(p, sc, want_w, &V, &Cinv);
  if (rc) return rc;
  void* tmp = nullptr;
  T *mbar = nullptr, *mean_d = nullptr;
  if (want_mbar) { CK(sc.alloc(&tmp, (size_t)n_pad * sizeof(T))); mbar = (T*)tmp; CK(cudaMemsetAsync(mbar, 0, (size_t)n_pad * sizeof(T), s)); }
  if (mean->kind == 2) { rc = upload<T>(ctx, sc, mean->v, N, true, &mean_d); if (rc) return rc; }
  rc = weighted_cols_pullback<T>(ctx, sc, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, V, N, Y, mean->kind, mean->c,
                                 mean_d, S, lp_bar, true, Cinv, mbar, y_bar_out, nullptr);
  if (rc) return rc;
  if (want_w) {
    CK(sc.alloc(&tmp, (size_t)n_pad * sizeof(T)));
    T* zero_alpha = (T*)tmp;
    CK(cudaMemsetAsync(zero_alpha, 0, (size_t)n_pad * sizeof(T), s));
    rc = grad_reductions<T>(p, sc, Cinv, zero_alpha, grad_out, noise_diag_out, layout, x_grad_out);
    if (rc) return rc;
  }
  if (want_mbar) {
    rc = download<T>(ctx, mean_diag_out, mbar, (size_t)N, false);
    if (rc) return rc;
  }
  if (grad_out) {  // d/d ConstMean c = sum_i mbar_i
    rc = host_sum<T>(ctx, mbar, N, &grad_out[4]);
    if (rc) return rc;
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// extra product columns of the posterior gradients' blocks: [.. alpha], [.. mubar], the -beta' row (one used, 16 keeps
// alignment)
constexpr int64_t POST_XK = 16;

// The training side shared by agp_post_pred_logpdf_grad and agp_post_rand_grad, from the test side's cotangents.  On
// entry: Ws (m_pad x (m_pad + POST_XK)) holds -2 Sigmabar in both triangles of its first m_pad columns and mubar in
// column m_pad, zero elsewhere; P (n_pad x (m_pad + POST_XK)) holds P = C^-1 K_xs in its first m_pad columns (padding
// rows and columns zero).  The tail puts alpha into column m_pad of P, forms beta = P mubar (ybar = beta, mbar = -beta)
// and, with want_red, the stacked W over [x; x*] (the comment of post_pred_logpdf_grad_impl) and its reductions, split
// into the training and the test outputs; grad_out[3] and [4] are the training noise and the ConstMean entries.
template <typename T>
int post_pred_tail(agp_post* p, Scratch& sc, int layout, const T* Xst, int64_t M, const T* Ws, T* P, bool want_red,
                   double* grad_out, void* noise_diag_out, void* mean_diag_out, void* y_bar_out, void* x_grad_out,
                   void* noise_s_diag_out, void* xs_grad_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  const int64_t N = p->n, n_pad = p->n_pad, m_pad = round_up(M, TILE);
  const int D = p->D;
  constexpr int64_t XK = POST_XK;
  const T* mubar = Ws + m_pad * m_pad;
  const cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  void* tmp = nullptr;
  int rc = AGP_OK;
  CK(cudaMemsetAsync(P + n_pad * m_pad, 0, (size_t)n_pad * XK * sizeof(T), s));
  CK(cudaMemcpyAsync(P + n_pad * m_pad, p->alpha, (size_t)N * sizeof(T), cudaMemcpyDeviceToDevice, s));
  CK(sc.alloc(&tmp, (size_t)n_pad * 2 * sizeof(T)));
  T* beta = (T*)tmp;
  T* nbeta = beta + n_pad;
  CK(cudaMemsetAsync(beta, 0, (size_t)n_pad * 2 * sizeof(T), s));
  launch_gemv_n_acc<T>(P, n_pad, N, M, mubar, beta, s);
  CK(cudaMemcpyAsync(nbeta, beta, (size_t)n_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
  launch_scale<T>(nbeta, n_pad, -1.0, s);
  rc = download<T>(ctx, y_bar_out, beta, (size_t)N, false);
  if (rc) return rc;
  rc = download<T>(ctx, mean_diag_out, nbeta, (size_t)N, false);
  if (rc) return rc;
  if (want_red) {
    const int64_t Lst = n_pad + m_pad, ldw = Lst + XK;
    CK(sc.alloc(&tmp, (size_t)ldw * Lst * sizeof(T)));
    T* Wst = (T*)tmp;
    {
      GemmArgs g{};  // -Kbar_sx = -[Ws mubar][P alpha]' into rows n_pad.. of the first n_pad columns
      g.A = Ws; g.lda = m_pad; g.a_kmajor = 0;
      g.B = P; g.ldb = n_pad; g.b_kmajor = 0;
      g.C = Wst + n_pad; g.ldc = ldw; g.M = m_pad; g.N = n_pad; g.K = m_pad + XK; g.alpha_neg = 1;
      launch_gemm<T>(g, s);
    }
    CK(cudaMemset2DAsync(Wst + Lst, (size_t)ldw * sizeof(T), 0, (size_t)XK * sizeof(T), (size_t)n_pad, s));
    CK(cudaMemcpy2DAsync(Wst + Lst, (size_t)ldw * sizeof(T), nbeta, sizeof(T), sizeof(T), (size_t)n_pad,
                         cudaMemcpyDeviceToDevice, s));  // the -beta' row under -Kbar_sx
    {
      GemmArgs g{};  // -2 Cbar = -[P alpha][-Kbar_sx; -beta'], lower tiles
      g.A = P; g.lda = n_pad; g.a_kmajor = 0;
      g.B = Wst + n_pad; g.ldb = ldw; g.b_kmajor = 1;
      g.C = Wst; g.ldc = ldw; g.M = n_pad; g.N = n_pad; g.K = m_pad + XK; g.alpha_neg = 1; g.lower_only = 1;
      launch_gemm<T>(g, s);
    }
    launch_copy2d<T>(Ws, m_pad, Wst + n_pad + n_pad * ldw, ldw, m_pad, m_pad, s);  // -2 Sigmabar
    CK(sc.alloc(&tmp, (size_t)Lst * (D + 1) * sizeof(T)));
    T* Xcat = (T*)tmp;  // [x; x*] point-major, then alpha = 0
    T* zalpha = Xcat + Lst * D;
    CK(cudaMemcpyAsync(Xcat, p->Xt, (size_t)n_pad * D * sizeof(T), cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(Xcat + n_pad * D, Xst, (size_t)m_pad * D * sizeof(T), cudaMemcpyDeviceToDevice, s));
    CK(cudaMemsetAsync(zalpha, 0, (size_t)Lst * sizeof(T), s));
    const bool want_diag = grad_out || noise_diag_out || noise_s_diag_out;
    const bool want_x = x_grad_out || xs_grad_out;
    T *nd = nullptr, *xg = nullptr;
    if (want_diag) { CK(sc.alloc(&tmp, (size_t)Lst * sizeof(T))); nd = (T*)tmp; }
    if (want_x) { CK(sc.alloc(&tmp, (size_t)Lst * D * sizeof(T))); xg = (T*)tmp; }
    const bool saved = ctx->out_dev_override;
    ctx->out_dev_override = true;  // the stacked outputs stay on the device and are split below
    rc = grad_reductions_on<T>(p, sc, Xcat, Lst, Lst, Wst, ldw, zalpha, grad_out, nd, layout, xg);
    ctx->out_dev_override = saved;
    if (rc) return rc;
    rc = download<T>(ctx, noise_diag_out, nd, (size_t)N, false);
    if (rc) return rc;
    rc = download<T>(ctx, noise_s_diag_out, want_diag ? nd + n_pad : nullptr, (size_t)M, false);
    if (rc) return rc;
    // the stacked input gradient in `layout`: point-major rows [0, N) and [n_pad, n_pad + M); feature-major columns
    auto split_x = [&](void* out, int64_t off, int64_t cnt) -> int {
      if (!out) return AGP_OK;
      if (layout == AGP_POINT_MAJOR)
        CK(cudaMemcpyAsync(out, xg + off * D, (size_t)cnt * D * sizeof(T), kout, s));
      else
        CK(cudaMemcpy2DAsync(out, (size_t)cnt * sizeof(T), xg + off, (size_t)Lst * sizeof(T), (size_t)cnt * sizeof(T),
                             (size_t)D, kout, s));
      return AGP_OK;
    };
    rc = split_x(x_grad_out, 0, N);
    if (rc) return rc;
    rc = split_x(xs_grad_out, n_pad, M);
    if (rc) return rc;
    if (grad_out) {  // d/d sigma^2 = sum_i Cbar_ii and d/d ConstMean c = sum mubar - sum beta
      double sn = 0.0, sm = 0.0, sb = 0.0;
      rc = host_sum<T>(ctx, nd, N, &sn); if (rc) return rc;
      rc = host_sum<T>(ctx, beta, N, &sb); if (rc) return rc;
      rc = host_sum<T>(ctx, mubar, M, &sm); if (rc) return rc;
      grad_out[3] = sn;
      grad_out[4] = sm - sb;
    }
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// ---- pullback of F = sum_s w_s logpdf(posterior(fx, y)(x*, Sigma*), Y*[:, s]) on a handle from agp_fit (agp.h
// agp_post_pred_logpdf_grad).  With C = L L', alpha = C^-1 delta, A = L^-1 K_xs, P = C^-1 K_xs = V'A (V = L^-1),
// mu* = m* + K_sx alpha, Sigma = K_ss - A'A + Sigma* = L* L*' and E = Y* - mu* 1':
//   -2 Sigmabar = (sum w) Sigma^-1 - B diag(w) B',  B = Sigma^-1 E   (chunks of up to 1024 columns, as in the _cols
//                 gradient, into the lower and upper tiles of one m_pad x m_pad buffer Ws),  mubar = B w,  Ybar* = -B diag(w)
//   -Kbar_sx    = -[Ws mubar] [P alpha]'          (tile GEMM, K = m_pad + 1)
//   -2 Cbar     = P Kbar_sx + alpha beta' = -[P alpha] [-Kbar_sx; -beta']   (lower tiles, K = m_pad + 1),  beta = P mubar
// The three blocks are the lower triangle of one symmetric W over the stacked points [x (n_pad rows); x* (m_pad rows)]:
// the objective's kernel terms are <Cbar, K_xx> + <Kbar_sx, K_sx> + <Sigmabar, K_ss> = 1/2 <W, K([x; x*])> with
// W = [2 Cbar, Kbar_xs; Kbar_sx, 2 Sigmabar], so grad_reductions_on with alpha = 0 and -W in place of C^-1 gives the
// hyper-parameters, the noise diagonals (1/2 W_ii: Cbar_ii, then Sigmabar_mm) and both input gradients in one pass of
// the existing reductions.  Padding rows of either block have zero rows and columns in W and add nothing.  The -beta'
// row sits in XK extra rows under the stacked buffer so that the K = m_pad + 1 product reads it from the same operand.
// Why this and not a rectangular reduction over Kbar_sx (or, for single kernels, vfe_cross_grad_kernel +
// vfe_x_grad_kernel with isn = 1, delta = alpha, r = mubar): the stacked pass visits the same pairs, N^2/2 + NM + M^2/2,
// with kernels that are already validated for every family, transform and composite descriptor, both dtypes and both
// layouts, so it needs no new kernel, no float instantiation of the VFE ones and no second copy of the composite
// derivative rules; the VFE kernels take the square sums only from their own K_zz pass and would still need grad_x and
// grad_reduce for K_xx and K_ss.  Its cost is memory: the stacked buffer holds the 2 NM elements of the unused upper block
// besides the blocks.  V, A, the factor of Sigma and Vs are freed before it is allocated, so the peak is about
// (N + M)^2 + NM + M^2 elements of T (W, P, Ws) besides the handle (agp.h).
template <typename T>
int post_pred_logpdf_grad_impl(agp_post* p, int layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                               const agp_noise* noise_s, const void* Ys, int S, const double* lp_bar, void* lp_out,
                               double* grad_out, void* noise_diag_out, void* mean_diag_out, void* y_bar_out, void* x_grad_out,
                               void* noise_s_diag_out, void* mean_s_diag_out, void* ys_bar_out, void* xs_grad_out) {
  agp_ctx* ctx = p->ctx;
  if (S < 1) { ctx->err = "S must be >= 1"; return AGP_ERR_INVALID; }
  if (!Ys) { ctx->err = "Ys is NULL"; return AGP_ERR_INVALID; }
  if (!Xs) { ctx->err = "Xs is NULL"; return AGP_ERR_INVALID; }
  if (M <= 0) { ctx->err = "M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  agp_mean mz;
  int rc = post_side_defaults(p, &mean_s, &noise_s, &mz);
  if (rc) return rc;
  rc = logpdf_grad_prelude<T>(p, layout);
  if (rc) return rc;
  cudaStream_t s = ctx->stream;
  const int64_t n_pad = p->n_pad, m_pad = round_up(M, TILE), ldf = m_pad + TILE;
  const int nblk = (int)(m_pad / TILE);
  constexpr int64_t XK = POST_XK;
  const bool want_red = grad_out || noise_diag_out || x_grad_out || noise_s_diag_out || xs_grad_out;
  const bool want_beta = want_red || mean_diag_out || y_bar_out;
  Scratch sc(ctx);
  void* tmp = nullptr;

  // ---- forward: mu*, A = L^-1 K_xs, Sigma = K_ss + Sigma* - A'A and its factor
  T *Xst = nullptr, *A = nullptr;
  rc = post_cross<T>(p, sc, layout, Xs, M, m_pad, &Xst, &A);
  if (rc) return rc;
  T *mean_d = nullptr, *noise_d = nullptr;
  if (mean_s->kind == 2) { rc = upload<T>(ctx, sc, mean_s->v, M, true, &mean_d); if (rc) return rc; }
  if (noise_s->kind == 1) { rc = upload<T>(ctx, sc, noise_s->v, M, true, &noise_d); if (rc) return rc; }
  CK(sc.alloc(&tmp, (size_t)m_pad * sizeof(T)));
  T* mu = (T*)tmp;
  CK(cudaMemsetAsync(mu, 0, (size_t)m_pad * sizeof(T), s));
  launch_gemv_t<T>(A, n_pad, n_pad, M, (const T*)p->alpha, mean_s->kind, mean_s->c, mean_d, mu, s);
  forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, A, n_pad, m_pad);
  T *Lf = nullptr, *Dinv = nullptr;
  double* dscal = nullptr;
  int* dinfo = nullptr;
  rc = post_cov_factor<T>(p, sc, Xst, A, M, noise_s, noise_d, (const T*)nullptr, 0, mu, &Lf, &Dinv, &dscal, &dinfo);
  if (rc) return rc;
  rc = post_cov_status(ctx, dinfo);
  if (rc) return rc;
  double logdet = 0.0;
  rc = host_sum<double>(ctx, dscal, nblk, &logdet);
  if (rc) return rc;
  logdet *= 2.0;

  // ---- Sigma^-1 = Vs'Vs (Vs = L*^-1 with its identity padding zeroed, so nothing outside M x M is nonzero), then the
  // columns: Ws = -2 Sigmabar, mubar (column m_pad of Ws), Ybar*, and the squared Mahalanobis norms for the values
  CK(sc.alloc(&tmp, (size_t)m_pad * m_pad * sizeof(T)));
  T* Vs = (T*)tmp;
  CK(cudaMemsetAsync(Vs, 0, (size_t)m_pad * m_pad * sizeof(T), s));
  launch_add_diag<T>(Vs, m_pad, M, 1.0, s);
  forward_subst_multi<T>(ctx, (const T*)Lf, ldf, (const T*)Dinv, m_pad, Vs, m_pad, m_pad);
  CK(sc.alloc(&tmp, (size_t)m_pad * (m_pad + XK) * sizeof(T)));
  T* Ws = (T*)tmp;
  T* mubar = Ws + m_pad * m_pad;
  CK(cudaMemsetAsync(Ws, 0, (size_t)m_pad * (m_pad + XK) * sizeof(T), s));
  if (want_red) {
    GemmArgs g{};  // Sigma^-1, both triangles
    g.A = Vs; g.lda = m_pad; g.a_kmajor = 1;
    g.B = Vs; g.ldb = m_pad; g.b_kmajor = 1;
    g.C = Ws; g.ldc = m_pad; g.M = m_pad; g.N = m_pad; g.K = m_pad;
    launch_gemm<T>(g, s);
  }
  CK(sc.alloc(&tmp, (size_t)S * sizeof(T)));
  T* sq = (T*)tmp;
  CK(cudaMemsetAsync(sq, 0, (size_t)S * sizeof(T), s));
  rc = weighted_cols_pullback<T>(ctx, sc, (const T*)Lf, ldf, (const T*)Dinv, m_pad, Vs, M, Ys, 2, 0.0, mu, S, lp_bar,
                                 false, want_red ? Ws : nullptr, mubar, ys_bar_out, sq);
  if (rc) return rc;
  if (lp_out) {  // logpdf_s = -1/2 (M log 2 pi + logdet Sigma + |L*^-1 e_s|^2)
    std::vector<T> h((size_t)S);
    CK(cudaMemcpyAsync(h.data(), sq, (size_t)S * sizeof(T), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const double log2pi = 1.8378770664093454835606594728112;
    for (int j = 0; j < S; ++j) h[(size_t)j] = (T)(-0.5 * ((double)M * log2pi + logdet + (double)h[(size_t)j]));
    CK(cudaMemcpyAsync(lp_out, h.data(), (size_t)S * sizeof(T),
                       ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyHostToDevice : cudaMemcpyHostToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  rc = download<T>(ctx, mean_s_diag_out, mubar, (size_t)M, false);
  if (rc) return rc;
  // buffers are returned to the pool as soon as they are dead (stream-ordered), so that V and the stacked W are never
  // live together
  auto drop = [&](void* q) { sc.release(q); cudaFreeAsync(q, s); };
  drop(Vs); drop(Lf); drop(Dinv);

  // ---- training side: P = V'A, then the blocks and the reductions (post_pred_tail)
  if (want_beta) {
    T *V = nullptr, *unused = nullptr;
    rc = inverse_factor<T>(p, sc, false, &V, &unused);
    if (rc) return rc;
    CK(sc.alloc(&tmp, (size_t)n_pad * (m_pad + XK) * sizeof(T)));
    T* P = (T*)tmp;
    {
      GemmArgs g{};
      g.A = V; g.lda = n_pad; g.a_kmajor = 1;
      g.B = A; g.ldb = n_pad; g.b_kmajor = 1;
      g.C = P; g.ldc = n_pad; g.M = n_pad; g.N = m_pad; g.K = n_pad;
      launch_gemm<T>(g, s);
    }
    drop(V); drop(A);
    rc = post_pred_tail<T>(p, sc, layout, Xst, M, Ws, P, want_red, grad_out, noise_diag_out, mean_diag_out, y_bar_out,
                           x_grad_out, noise_s_diag_out, xs_grad_out);
    if (rc) return rc;
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

template <typename T>
int post_solve_lower_impl(agp_post* p, const void* Bh, int64_t nrhs, void* V_out) {
  agp_ctx* ctx = p->ctx;
  { int rrc = post_replicate<T>(p); if (rrc) return rrc; }
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (nrhs <= 0) return AGP_OK;
  const int64_t c_pad = round_up(nrhs, 4);
  Scratch sc(ctx);
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)p->n_pad * c_pad * sizeof(T)));
  T* B = (T*)tmp;
  CK(cudaMemsetAsync(B, 0, (size_t)p->n_pad * c_pad * sizeof(T), s));
  cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  int64_t off = 0;
  for (auto& sg : p->segs) {  // compact rows -> padded row positions
    CK(cudaMemcpy2DAsync(B + sg.first, (size_t)p->n_pad * sizeof(T), (const T*)Bh + off, (size_t)p->n * sizeof(T),
                         (size_t)sg.second * sizeof(T), (size_t)nrhs, kin, s));
    off += sg.second;
  }
  forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, p->n_pad, B, p->n_pad, c_pad);
  off = 0;
  for (auto& sg : p->segs) {
    CK(cudaMemcpy2DAsync((T*)V_out + off, (size_t)p->n * sizeof(T), B + sg.first, (size_t)p->n_pad * sizeof(T),
                         (size_t)sg.second * sizeof(T), (size_t)nrhs, kout, s));
    off += sg.second;
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

template <typename T>
int post_export_impl(agp_post* p, void* U_out) {
  agp_ctx* ctx = p->ctx;
  { int rrc = post_replicate<T>(p); if (rrc) return rrc; }
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  Scratch sc(ctx);
  void* tmp = nullptr;
  const int64_t* map_d = nullptr;
  if (p->segs.size() > 1) {  // extended posterior: valid rows are not contiguous
    std::vector<int64_t> map;
    for (auto& sg : p->segs) for (int64_t i = 0; i < sg.second; ++i) map.push_back(sg.first + i);
    CK(sc.alloc(&tmp, map.size() * sizeof(int64_t)));
    CK(cudaMemcpyAsync(tmp, map.data(), map.size() * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    map_d = (const int64_t*)tmp;
  }
  T* Ud = (T*)U_out;
  if (ctx->memspace != AGP_MEM_DEVICE) {
    CK(sc.alloc(&tmp, (size_t)p->n * p->n * sizeof(T)));
    Ud = (T*)tmp;
  }
  if (map_d) launch_export_upper_map<T>((const T*)p->L, p->lda, p->n, map_d, Ud, p->n, s);
  else launch_export_upper<T>((const T*)p->L, p->lda, p->n, Ud, p->n, s);
  if (ctx->memspace != AGP_MEM_DEVICE)
    CK(cudaMemcpyAsync(U_out, Ud, (size_t)p->n * p->n * sizeof(T), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// ---- sequential conditioning: posterior(fx::FiniteGP{<:PosteriorGP}, y) via update_chol
// (/root/reference/src/exact_gpr_posterior.jl:46-56, /root/reference/src/util/common_covmat_ops.jl:38-42).
// L21 = C21 L11^-T by the same panel solves the factorisation uses (one per old column block), then
// ONE long-K trailing update C22 -= L21 L21', then a Cholesky of the new diagonal part.  The border
// rows carry [delta1; delta2]' through all of it, so v = L^-1 delta comes out of the same kernels.
template <typename T>
int post_extend_impl(agp_post* p, int layout, const void* X2, int64_t N2, const void* y2, const agp_mean* mean2,
                     const agp_noise* noise2, void* alpha_out, agp_post** post_out) {
  agp_ctx* ctx = p->ctx;
  { int rrc = post_replicate<T>(p); if (rrc) return rrc; }
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (N2 <= 0) { ctx->err = "N2 must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (!X2 || !y2) { ctx->err = "X2/y2 is NULL"; return AGP_ERR_INVALID; }
  static const agp_mean zero_mean{0, 0.0, nullptr};
  static const agp_noise default_noise{0, 1e-18, nullptr};
  if (!mean2) mean2 = &zero_mean;
  if (!noise2) noise2 = &default_noise;
  Scratch sc(ctx);
  const int64_t n1p = p->n_pad, n2p = round_up(N2, TILE), np = n1p + n2p, ldn = np + TILE;
  const int nblk1 = (int)(n1p / TILE), nblk2 = (int)(n2p / TILE), nblk = nblk1 + nblk2;
  const int D = p->D;
  T *mean_d = nullptr, *noise_d = nullptr, *y2d = nullptr, *X2t = nullptr;
  int rc;
  if (mean2->kind == 2) { rc = upload<T>(ctx, sc, mean2->v, N2, true, &mean_d); if (rc) return rc; }
  if (noise2->kind == 1) { rc = upload<T>(ctx, sc, noise2->v, N2, true, &noise_d); if (rc) return rc; }
  rc = upload<T>(ctx, sc, y2, N2, false, &y2d); if (rc) return rc;
  rc = prep_points<T>(ctx, sc, &p->k, (const T*)p->ard, layout, X2, N2, n2p, D, &X2t, false); if (rc) return rc;

  void *Ln = nullptr, *Dn = nullptr, *Xn = nullptr, *an = nullptr, *dn = nullptr, *vn = nullptr;
  CK(cudaMallocAsync(&Ln, (size_t)ldn * np * sizeof(T), s));
  CK(cudaMallocAsync(&Dn, (size_t)nblk * TILE * TILE * sizeof(T), s));
  CK(cudaMallocAsync(&Xn, (size_t)np * D * sizeof(T), s));
  CK(cudaMallocAsync(&an, (size_t)np * sizeof(T), s));
  CK(cudaMallocAsync(&dn, (size_t)np * sizeof(T), s));
  CK(cudaMallocAsync(&vn, (size_t)np, s));
  T* L = (T*)Ln; T* Dinv = (T*)Dn;
  unsigned char* valid = (unsigned char*)vn;
  // carry the old state over
  launch_copy2d<T>((const T*)p->L, p->lda, L, ldn, n1p, n1p, s);
  CK(cudaMemcpyAsync(Dinv, p->Dinv, (size_t)nblk1 * TILE * TILE * sizeof(T), cudaMemcpyDeviceToDevice, s));
  CK(cudaMemcpyAsync(Xn, p->Xt, (size_t)n1p * D * sizeof(T), cudaMemcpyDeviceToDevice, s));
  CK(cudaMemcpyAsync((T*)Xn + n1p * D, X2t, (size_t)n2p * D * sizeof(T), cudaMemcpyDeviceToDevice, s));
  if (p->valid) CK(cudaMemcpyAsync(valid, p->valid, (size_t)n1p, cudaMemcpyDeviceToDevice, s));
  else { CK(cudaMemsetAsync(valid, 1, (size_t)p->n, s)); CK(cudaMemsetAsync(valid + p->n, 0, (size_t)(n1p - p->n), s)); }
  CK(cudaMemsetAsync(valid + n1p, 1, (size_t)N2, s));
  CK(cudaMemsetAsync(valid + n1p + N2, 0, (size_t)(n2p - N2), s));
  CK(cudaMemcpyAsync(dn, p->delta, (size_t)n1p * sizeof(T), cudaMemcpyDeviceToDevice, s));
  CK(cudaMemsetAsync((T*)dn + n1p, 0, (size_t)n2p * sizeof(T), s));
  launch_sub_mean<T>(y2d, N2, mean2->kind, mean2->c, mean_d, (T*)dn + n1p, s);
  // C21 = K(x2, x1) and C22 = K(x2, x2) + Sigma_y2 straight into the new factor buffer
  GramParams g21{};
  fill_gram_params<T>(g21, &p->k, 0, 0, N2, p->n, nullptr, nullptr, p->comp);
  g21.mask_b = valid;  // old rows (first n1p entries of the new mask)
  launch_gram<T>(X2t, (const T*)Xn, n2p, n1p, D, L + n1p, ldn, g21, s);
  GramParams g22{};
  fill_gram_params<T>(g22, &p->k, 1, 1, N2, N2, noise2, noise_d, p->comp);
  launch_gram<T>(X2t, X2t, n2p, n2p, D, L + n1p + n1p * ldn, ldn, g22, s);
  launch_border_init<T>(L, ldn, np, np, (const T*)dn, np, 1, 0, 0.0, (const T*)nullptr, s);
  // panel solves of the new rows (+ border) against the old factor
  const int64_t Mr = n2p + TILE;
  for (int k = 0; k < nblk1; ++k) {
    T* Rk = L + n1p + (int64_t)k * TILE * ldn;
    GemmArgs t{};
    t.A = Rk; t.lda = ldn; t.B = Dinv + (int64_t)k * TILE * TILE; t.ldb = TILE;
    t.C = Rk; t.ldc = ldn; t.M = Mr; t.N = TILE; t.K = TILE;
    launch_gemm<T>(t, s);
    const int64_t cols_rest = n1p - (int64_t)(k + 1) * TILE;
    if (cols_rest <= 0) continue;
    GemmArgs u{};
    u.A = Rk; u.lda = ldn;
    u.B = L + (int64_t)(k + 1) * TILE + (int64_t)k * TILE * ldn; u.ldb = ldn;
    u.C = Rk + (int64_t)TILE * ldn; u.ldc = ldn; u.M = Mr; u.N = cols_rest; u.K = TILE; u.alpha_neg = 1; u.beta_one = 1;
    launch_gemm<T>(u, s);
  }
  {  // C22 -= L21 L21'  (one launch, K = n1p)
    GemmArgs u{};
    u.A = L + n1p; u.lda = ldn; u.B = L + n1p; u.ldb = ldn;
    u.C = L + n1p + n1p * ldn; u.ldc = ldn; u.M = Mr; u.N = n2p; u.K = n1p; u.alpha_neg = 1; u.beta_one = 1; u.lower_only = 1;
    launch_gemm<T>(u, s);
  }
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)(nblk2 + TILE + 2) * sizeof(double)));
  double* dscal = (double*)tmp;
  CK(sc.alloc(&tmp, sizeof(int)));
  int* dinfo = (int*)tmp;
  CK(cudaMemsetAsync(dinfo, 0, sizeof(int), s));
  CK(sc.alloc(&tmp, (size_t)(nblk + 1) * sizeof(int)));
  int* dflags = (int*)tmp;
  CK(sc.alloc(&tmp, (size_t)np * sizeof(T)));
  T* rwork = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)TILE * sizeof(T)));
  T* lp_d = (T*)tmp;
  prof_begin(ctx);
  cholesky_inplace<T>(ctx, L + n1p + n1p * ldn, ldn, n2p, n2p + TILE, Dinv + (int64_t)nblk1 * TILE * TILE, dscal, dinfo);
  launch_extract_v<T>(L, ldn, np, 1, rwork, dscal + nblk2, s);
  launch_bwd_solve<T>(L, ldn, Dinv, nblk, rwork, dflags, s);
  CK(cudaMemcpyAsync(an, rwork, (size_t)np * sizeof(T), cudaMemcpyDeviceToDevice, s));
  launch_finalize_logpdf<T>(dscal, nblk2, dscal + nblk2, 1, N2, lp_d, dscal + nblk2 + TILE, s);
  int h_info = 0;
  double h_ld = 0.0;
  CK(cudaMemcpyAsync(&h_info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&h_ld, dscal + nblk2 + TILE, sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (h_info != 0) {
    cudaFreeAsync(Ln, s); cudaFreeAsync(Dn, s); cudaFreeAsync(Xn, s); cudaFreeAsync(an, s); cudaFreeAsync(dn, s); cudaFreeAsync(vn, s);
    ctx->info = p->n + h_info;
    ctx->err = "extended covariance is not positive definite";
    return AGP_ERR_NOT_POSDEF;
  }
  if (post_out) {  // the reference's semantics: a NEW posterior, the conditioned-on one stays valid
    agp_post* q = new agp_post(*p);
    q->ard = nullptr;
    if (p->ard) {
      cudaMallocAsync(&q->ard, (size_t)D * sizeof(T), s);
      cudaMemcpyAsync(q->ard, p->ard, (size_t)D * sizeof(T), cudaMemcpyDeviceToDevice, s);
    }
    if (p->comp) {  // the new handle owns its own copy of the descriptor
      q->comp = new CompState(*p->comp);
      const size_t wb = p->comp->w.size() * sizeof(T);
      void* wd = nullptr;
      cudaMallocAsync(&wd, wb, s);
      cudaMemcpyAsync(wd, p->comp->desc.w, wb, cudaMemcpyDeviceToDevice, s);
      q->comp->desc.w = wd;
      q->comp->owns_w = true;
    }
    *post_out = q;
    p = q;
  } else {  // in place: the old state is released
    cudaFreeAsync(p->L, s); cudaFreeAsync(p->Dinv, s); cudaFreeAsync(p->Xt, s); cudaFreeAsync(p->alpha, s);
    cudaFreeAsync(p->delta, s);
    if (p->valid) cudaFreeAsync(p->valid, s);
  }
  p->L = Ln; p->Dinv = Dn; p->Xt = Xn; p->alpha = an; p->delta = dn; p->valid = valid;
  p->segs.push_back({n1p, N2});
  p->n += N2; p->n_pad = np; p->lda = ldn; p->logdet += h_ld;
  if (alpha_out) {
    int64_t off = 0;
    cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    for (auto& sg : p->segs) {
      CK(cudaMemcpyAsync((T*)alpha_out + off, (const T*)p->alpha + sg.first, (size_t)sg.second * sizeof(T), kout, s));
      off += sg.second;
    }
    CK(cudaStreamSynchronize(s));
  }
  return AGP_OK;
}

template <typename T>
int rand_impl(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout,
              const void* X, int64_t N, int D, const void* Z, int S, void* out) {
  if (S <= 0) return AGP_OK;
  if (!Z || !out) { ctx->err = "Z/out is NULL"; return AGP_ERR_INVALID; }
  Scratch outer(ctx);
  T* L = nullptr;
  int64_t lda = 0;
  int rc = fit_impl<T>(ctx, k, mean, noise, layout, X, N, D, nullptr, 0, nullptr, nullptr, nullptr, &L, &lda, &outer);
  if (rc) return rc;
  cudaStream_t s = ctx->stream;
  const int64_t n_pad = round_up(N, TILE), s_pad = round_up(S, 4);
  void* tmp = nullptr;
  CK(outer.alloc(&tmp, (size_t)n_pad * s_pad * sizeof(T) * 2));
  T* Zd = (T*)tmp; T* Od = Zd + n_pad * s_pad;
  CK(cudaMemsetAsync(Zd, 0, (size_t)n_pad * s_pad * sizeof(T), s));
  cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  CK(cudaMemcpy2DAsync(Zd, (size_t)n_pad * sizeof(T), Z, (size_t)N * sizeof(T), (size_t)N * sizeof(T), (size_t)S, kin, s));
  GemmArgs g{};  // out = L * Z (TRMM, lower)
  g.A = L; g.lda = lda; g.a_kmajor = 0;
  g.B = Zd; g.ldb = n_pad; g.b_kmajor = 1;
  g.C = Od; g.ldc = n_pad; g.M = n_pad; g.N = s_pad; g.K = n_pad; g.trmm_lower = 1;
  launch_gemm<T>(g, s);
  static const agp_mean zero_mean{0, 0.0, nullptr};
  if (!mean) mean = &zero_mean;
  T* mean_d = nullptr;
  if (mean->kind == 2) { rc = upload<T>(ctx, outer, mean->v, N, true, &mean_d); if (rc) return rc; }
  launch_add_mean_cols<T>(Od, n_pad, N, S, mean->kind, mean->c, mean_d, s);
  cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  CK(cudaMemcpy2DAsync(out, (size_t)N * sizeof(T), Od, (size_t)n_pad * sizeof(T), (size_t)N * sizeof(T), (size_t)S, kout, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// The pullback of a Cholesky sample out = L Z (C = L L', n rows, n_pad padded, L of leading dimension lda) at its
// cotangent Obar, shared by agp_rand_grad and agp_post_rand_grad.  Od and Zd hold Obar and Z (n_pad x s_pad, padding
// zeroed).  Into the caller's buffers:
//   Zb = L' Obar;  rowsum_i = sum_s Obar_is (fp64, in order);
//   and, when V = L^-1 (leading dimension n_pad) is given: Q = the lower triangle of Zb Z' mirrored, into Wout;
//   W1 = Q V, into Lt;  -V' W1 = -V'QV into Wout (its lower tiles only with lower_only, else both triangles).
// Lt (L', then W1) and Wout are n_pad x n_pad.  L' is taken whole from the factor (its storage above the diagonal blocks
// is not zeroed).
template <typename T>
void sample_pullback(agp_ctx* ctx, const T* L, int64_t lda, const T* V, int64_t n, int64_t n_pad, int S, int64_t s_pad,
                     const T* Od, const T* Zd, T* Zb, double* rowsum, T* Lt, T* Wout, bool lower_only) {
  cudaStream_t s = ctx->stream;
  launch_rowsum<T>(Od, n_pad, n, S, rowsum, s);
  launch_export_upper<T>(L, lda, n_pad, Lt, n_pad, s);
  {
    GemmArgs g{};
    g.A = Lt; g.lda = n_pad; g.a_kmajor = 0;
    g.B = Od; g.ldb = n_pad; g.b_kmajor = 1;
    g.C = Zb; g.ldc = n_pad; g.M = n_pad; g.N = s_pad; g.K = n_pad;
    launch_gemm<T>(g, s);
  }
  if (!V) return;
  {
    GemmArgs g{};  // Q = Zbar Z', lower tiles (K = S), then mirrored
    g.A = Zb; g.lda = n_pad; g.a_kmajor = 0;
    g.B = Zd; g.ldb = n_pad; g.b_kmajor = 0;
    g.C = Wout; g.ldc = n_pad; g.M = n_pad; g.N = n_pad; g.K = s_pad; g.lower_only = 1;
    launch_gemm<T>(g, s);
    launch_symmetrize_lower<T>(Wout, n_pad, n_pad, s);
  }
  {
    GemmArgs g{};  // W1 = Q V
    g.A = Wout; g.lda = n_pad; g.a_kmajor = 0;
    g.B = V; g.ldb = n_pad; g.b_kmajor = 1;
    g.C = Lt; g.ldc = n_pad; g.M = n_pad; g.N = n_pad; g.K = n_pad;
    launch_gemm<T>(g, s);
  }
  {
    GemmArgs g{};  // -V' W1
    g.A = V; g.lda = n_pad; g.a_kmajor = 1;
    g.B = Lt; g.ldb = n_pad; g.b_kmajor = 1;
    g.C = Wout; g.ldc = n_pad; g.M = n_pad; g.N = n_pad; g.K = n_pad; g.lower_only = lower_only ? 1 : 0; g.alpha_neg = 1;
    launch_gemm<T>(g, s);
  }
}

// ---- pullback of rand: out = m + L Z, C = K + Sigma_y = L L' (agp.h agp_rand_grad).  In fp64 whatever the caller's dtype
// (rand_grad_f32).  The factor comes from the factor-only fit as an agp_post, so the reductions of the logpdf gradient
// (grad_reductions) run on it with alpha = 0 and Cinv = -V'QV from sample_pullback (-2 Cbar, lower tiles).
// Three n_pad x n_pad buffers besides the factor; ~4 N^3 flop (the substitution N^3, Q V 2 N^3, the lower half of V'W1 N^3).
int rand_grad_f64(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout, const void* X,
                  int64_t N, int D, const void* Z, int S, const void* out_bar, double* grad_out, void* noise_diag_out,
                  void* mean_diag_out, void* x_grad_out, void* z_bar_out) {
  using T = double;
  agp_post* p = nullptr;
  int rc = fit_impl<T>(ctx, k, mean, noise, layout, X, N, D, nullptr, 0, nullptr, nullptr, &p, nullptr, nullptr, nullptr);
  if (rc) return rc;
  struct Guard { agp_post* p; ~Guard() { if (p) agp_post_free(p); } } guard{p};
  cudaStream_t s = ctx->stream;
  const int64_t n_pad = p->n_pad, s_pad = round_up(S, 4);
  Scratch sc(ctx);
  void* tmp = nullptr;
  const bool want_c = grad_out || noise_diag_out || x_grad_out;
  // the three N x N buffers first (fit_impl's note on the stream-ordered pool); V only when the reductions run
  CK(sc.alloc(&tmp, (size_t)n_pad * n_pad * sizeof(T)));
  T* B1 = (T*)tmp;  // L', then W1 = Q V
  CK(sc.alloc(&tmp, (size_t)n_pad * n_pad * sizeof(T)));
  T* B2 = (T*)tmp;  // Q, then -V'QV (lower tiles)
  T *V = nullptr, *unused = nullptr;
  if (want_c) { rc = inverse_factor<T>(p, sc, false, &V, &unused); if (rc) return rc; }
  CK(sc.alloc(&tmp, (size_t)n_pad * s_pad * sizeof(T) * 3));
  T* Od = (T*)tmp; T* Zd = Od + n_pad * s_pad; T* Zb = Zd + n_pad * s_pad;
  CK(sc.alloc(&tmp, (size_t)n_pad * sizeof(T)));
  T* zero_alpha = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)N * sizeof(double)));
  double* mbar = (double*)tmp;
  CK(cudaMemsetAsync(zero_alpha, 0, (size_t)n_pad * sizeof(T), s));
  CK(cudaMemsetAsync(Od, 0, (size_t)n_pad * s_pad * sizeof(T) * 2, s));  // zero padding rows / columns of Obar and Z
  const cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  const cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  if (S > 0) {
    CK(cudaMemcpy2DAsync(Od, (size_t)n_pad * sizeof(T), out_bar, (size_t)N * sizeof(T), (size_t)N * sizeof(T), (size_t)S, kin, s));
    CK(cudaMemcpy2DAsync(Zd, (size_t)n_pad * sizeof(T), Z, (size_t)N * sizeof(T), (size_t)N * sizeof(T), (size_t)S, kin, s));
  }
  // mbar_i = sum_s Obar_is, Zbar = L' Obar and, for the reductions, -V'QV = -2 Cbar (lower tiles) into B2
  sample_pullback<T>(ctx, (const T*)p->L, p->lda, V, N, n_pad, S, s_pad, Od, Zd, Zb, mbar, B1, B2, true);
  if (z_bar_out && S > 0)
    CK(cudaMemcpy2DAsync(z_bar_out, (size_t)N * sizeof(T), Zb, (size_t)n_pad * sizeof(T), (size_t)N * sizeof(T), (size_t)S, kout, s));
  if (want_c) {
    rc = grad_reductions<T>(p, sc, B2, zero_alpha, grad_out, noise_diag_out, layout, x_grad_out);
    if (rc) return rc;
  }
  rc = download<T>(ctx, mean_diag_out, mbar, (size_t)N, false);
  if (rc) return rc;
  if (grad_out) {  // d/d ConstMean c = sum_i mbar_i
    rc = host_sum<double>(ctx, mbar, N, &grad_out[4]);
    if (rc) return rc;
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

int rand_grad_check(agp_ctx* ctx, int layout, const void* X, const void* Z, int S, const void* out_bar) {
  int rc = check_layout(ctx, layout);
  if (rc) return rc;
  if (!X) { ctx->err = "X is NULL"; return AGP_ERR_INVALID; }
  if (S < 0) { ctx->err = "S must be >= 0"; return AGP_ERR_INVALID; }
  if (S > 0 && (!Z || !out_bar)) { ctx->err = "Z/out_bar is NULL"; return AGP_ERR_INVALID; }
  if (ctx->nccl) { ctx->err = "the gradient of rand runs on a single-GPU context"; return AGP_ERR_UNSUPPORTED; }
  return AGP_OK;
}

// An fp32 problem converted to fp64, for the gradients whose pullback runs in fp64 (rand_grad_f32, vfe_grad_f32).
// Parameter arrays are host memory (agp.h) and are widened on the host: the kernel's (the ARD values, or a composite's
// factors' ard and r), the mean and noise vectors (n points) and the jitter vector (m inducing points).  Point sets,
// targets and normals keep the caller's memory space: widened on the host, or cast into one fp64 scratch block on the
// device.  The fp64 outputs likewise, and narrow() rounds them into the caller's fp32 outputs.  Everything the converted
// problem points at lives as long as the object.
struct Fp64Problem {
  agp_ctx* ctx;
  bool dev;
  Scratch sc;
  std::vector<std::vector<double>> keep;  // widened host arrays
  agp_kernel k64{};
  agp_kernel_composite c64{};
  std::vector<agp_kernel_factor> f64;
  agp_mean m64{};
  agp_noise n64{}, j64{};
  const agp_mean* mean = nullptr;  // the converted parameters, NULL where the caller's are
  const agp_noise *noise = nullptr, *jitter = nullptr;
  struct Out { const double* src; void* dst; int64_t n; };
  std::vector<Out> outs;

  explicit Fp64Problem(agp_ctx* c) : ctx(c), dev(c->memspace == AGP_MEM_DEVICE), sc(c) {}

  const double* widen(const void* v, int64_t n) {
    if (!v) return nullptr;
    keep.emplace_back((size_t)n);
    for (int64_t i = 0; i < n; ++i) keep.back()[(size_t)i] = (double)((const float*)v)[i];
    return keep.back().data();
  }

  const agp_kernel* params(const agp_kernel* k, int D, const agp_mean* m_in, const agp_noise* n_in, int64_t n,
                          const agp_noise* j_in, int64_t m) {
    k64 = *k;
    if (k->family == AGP_COMPOSITE && k->composite) {
      c64 = *k->composite;
      int nf = 0;
      if (c64.nfactors && c64.nterms > 0 && c64.nterms <= AGP_COMP_MAX)
        for (int t = 0; t < c64.nterms; ++t) nf += c64.nfactors[t] > 0 ? c64.nfactors[t] : 0;
      if (c64.factors && nf <= AGP_COMP_MAX) {  // out-of-range descriptors are reported by comp_build
        f64.assign(c64.factors, c64.factors + nf);
        for (auto& f : f64) { f.ard = widen(f.ard, D); f.r = widen(f.r, D); }
        c64.factors = f64.data();
      }
      k64.composite = &c64;
    } else if (k->transform == AGP_T_ARD) {
      k64.ard = widen(k->ard, D);
    }
    if (m_in) { m64 = *m_in; if (m_in->kind == 2) m64.v = widen(m_in->v, n); mean = &m64; }
    if (n_in) { n64 = *n_in; if (n_in->kind == 1) n64.v = widen(n_in->v, n); noise = &n64; }
    if (j_in) { j64 = *j_in; if (j_in->kind == 1) j64.v = widen(j_in->v, m); jitter = &j64; }
    return &k64;
  }

  // fp64 copies of the fp32 arrays in (pointer, count); a NULL array stays NULL
  int inputs(std::initializer_list<std::pair<const void*, int64_t>> in, const double** out) {
    if (!dev) {
      for (const auto& a : in) *out++ = widen(a.first, a.second);
      return AGP_OK;
    }
    int64_t total = 0;
    for (const auto& a : in) total += a.second;
    void* tmp = nullptr;
    CK(sc.alloc(&tmp, (size_t)total * sizeof(double)));
    double* b = (double*)tmp;
    for (const auto& a : in) {
      *out = nullptr;
      if (a.first) { launch_cast<float, double>((const float*)a.first, b, a.second, ctx->stream); *out = b; }
      ++out;
      b += a.second;
    }
    return AGP_OK;
  }

  // fp64 buffers for the fp32 outputs in (pointer, count); NULL where the output is not asked for
  int outputs(std::initializer_list<std::pair<void*, int64_t>> o, double** out) {
    int64_t total = 0;
    for (const auto& a : o) if (a.first) total += a.second;
    double* b = nullptr;
    if (dev) { void* tmp = nullptr; CK(sc.alloc(&tmp, (size_t)total * sizeof(double))); b = (double*)tmp; }
    for (const auto& a : o) {
      *out = nullptr;
      if (a.first) {
        if (dev) { *out = b; b += a.second; }
        else { keep.emplace_back((size_t)a.second); *out = keep.back().data(); }
        outs.push_back(Out{*out, a.first, a.second});
      }
      ++out;
    }
    return AGP_OK;
  }

  int narrow() {
    for (const Out& o : outs) {
      if (o.n <= 0) continue;
      if (!dev) { for (int64_t i = 0; i < o.n; ++i) ((float*)o.dst)[i] = (float)o.src[i]; }
      else launch_cast<double, float>(o.src, (float*)o.dst, o.n, ctx->stream);
    }
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return AGP_OK;
  }
};

// fp32 problems: the pullback is formed on the problem converted to fp64 and its outputs rounded to fp32.  -V'QV carries
// terms of the order of cond(C) that cancel (agp.h).
int rand_grad_f32(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout, const void* X,
                  int64_t N, int D, const void* Z, int S, const void* out_bar, double* grad_out, void* noise_diag_out,
                  void* mean_diag_out, void* x_grad_out, void* z_bar_out) {
  int rc = check_kernel(ctx, k, D);
  if (rc) return rc;
  if (N <= 0) { ctx->err = "N must be positive"; return AGP_ERR_DIM_MISMATCH; }
  CK(cudaSetDevice(ctx->device));
  Fp64Problem p(ctx);
  const agp_kernel* k64 = p.params(k, D, mean, noise, N, nullptr, 0);
  const int64_t NS = N * (int64_t)S;
  const double* in[3];  // X, Z, out_bar
  rc = p.inputs({{X, N * D}, {Z, NS}, {out_bar, NS}}, in);
  if (rc) return rc;
  double* out[4];  // noise_diag, mean_diag, x_grad, z_bar
  rc = p.outputs({{noise_diag_out, N}, {mean_diag_out, N}, {x_grad_out, N * D}, {z_bar_out, NS}}, out);
  if (rc) return rc;
  rc = rand_grad_f64(ctx, k64, p.mean, p.noise, layout, in[0], N, D, in[1], S, in[2], grad_out, out[0], out[1],
                     out[2], out[3]);
  if (rc) return rc;
  return p.narrow();
}

// ---- pullback of rand(posterior(fx, y)(x*, Sigma*), S) on a handle from agp_fit (agp.h agp_post_rand_grad).  The forward
// is agp_post_rand's: mu* = m* + K_sx alpha, A = L^-1 K_xs, Sigma = K_ss + Sigma* - A'A = L* L*', out = mu* 1' + L* Z.
// The head is sample_pullback on L*: Zbar = L*' Obar, mubar = Obar 1 and -V*'QV* = -2 Sigmabar in both triangles
// (V* = L*^-1 with its identity padding zeroed, as in the held-out gradient).  From there the training side is the
// held-out gradient's (post_pred_tail), except that P = C^-1 K_xs = L^-T A comes from backward_subst_multi (N^2 M flop)
// instead of V = L^-1 (N^3) and V'A: no N x N buffer is allocated besides the stacked W, and the call has no N^3 term.
template <typename T>
int post_rand_grad_impl(agp_post* p, int layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                        const agp_noise* noise_s, const void* Z, int S, const void* out_bar, double* grad_out,
                        void* noise_diag_out, void* mean_diag_out, void* y_bar_out, void* x_grad_out, void* noise_s_diag_out,
                        void* mean_s_diag_out, void* z_bar_out, void* xs_grad_out) {
  agp_ctx* ctx = p->ctx;
  if (S < 1) { ctx->err = "S must be >= 1"; return AGP_ERR_INVALID; }
  if (!Z || !out_bar) { ctx->err = "Z/out_bar is NULL"; return AGP_ERR_INVALID; }
  if (!Xs) { ctx->err = "Xs is NULL"; return AGP_ERR_INVALID; }
  if (M <= 0) { ctx->err = "M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  agp_mean mz;
  int rc = post_side_defaults(p, &mean_s, &noise_s, &mz);
  if (rc) return rc;
  rc = logpdf_grad_prelude<T>(p, layout);
  if (rc) return rc;
  cudaStream_t s = ctx->stream;
  const int64_t n_pad = p->n_pad, m_pad = round_up(M, TILE), ldf = m_pad + TILE, s_pad = round_up(S, 4);
  constexpr int64_t XK = POST_XK;
  const bool want_red = grad_out || noise_diag_out || x_grad_out || noise_s_diag_out || xs_grad_out;
  const bool want_beta = want_red || mean_diag_out || y_bar_out;
  const cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  const cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  Scratch sc(ctx);
  void* tmp = nullptr;
  auto drop = [&](void* q) { sc.release(q); cudaFreeAsync(q, s); };

  // ---- forward: mu*, A = L^-1 K_xs, Sigma = K_ss + Sigma* - A'A and its factor (agp_post_rand's)
  T *Xst = nullptr, *A = nullptr;
  rc = post_cross<T>(p, sc, layout, Xs, M, m_pad, &Xst, &A);
  if (rc) return rc;
  T *mean_d = nullptr, *noise_d = nullptr;
  if (mean_s->kind == 2) { rc = upload<T>(ctx, sc, mean_s->v, M, true, &mean_d); if (rc) return rc; }
  if (noise_s->kind == 1) { rc = upload<T>(ctx, sc, noise_s->v, M, true, &noise_d); if (rc) return rc; }
  CK(sc.alloc(&tmp, (size_t)m_pad * sizeof(T)));
  T* mu = (T*)tmp;
  CK(cudaMemsetAsync(mu, 0, (size_t)m_pad * sizeof(T), s));
  launch_gemv_t<T>(A, n_pad, n_pad, M, (const T*)p->alpha, mean_s->kind, mean_s->c, mean_d, mu, s);
  forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, A, n_pad, m_pad);
  T *Lf = nullptr, *Dinv = nullptr;
  double* dscal = nullptr;
  int* dinfo = nullptr;
  rc = post_cov_factor<T>(p, sc, Xst, A, M, noise_s, noise_d, (const T*)nullptr, 0, mu, &Lf, &Dinv, &dscal, &dinfo);
  if (rc) return rc;
  rc = post_cov_status(ctx, dinfo);
  if (rc) return rc;

  // ---- head: Zbar, mubar (column m_pad of Ws) and, for the reductions, Ws = -2 Sigmabar
  CK(sc.alloc(&tmp, (size_t)m_pad * m_pad * sizeof(T)));
  T* Lt = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)m_pad * (m_pad + XK) * sizeof(T)));
  T* Ws = (T*)tmp;
  T* mubar = Ws + m_pad * m_pad;
  CK(cudaMemsetAsync(Ws, 0, (size_t)m_pad * (m_pad + XK) * sizeof(T), s));
  T* Vs = nullptr;
  if (want_red) {
    CK(sc.alloc(&tmp, (size_t)m_pad * m_pad * sizeof(T)));
    Vs = (T*)tmp;
    CK(cudaMemsetAsync(Vs, 0, (size_t)m_pad * m_pad * sizeof(T), s));
    launch_add_diag<T>(Vs, m_pad, M, 1.0, s);
    forward_subst_multi<T>(ctx, (const T*)Lf, ldf, (const T*)Dinv, m_pad, Vs, m_pad, m_pad);
  }
  CK(sc.alloc(&tmp, (size_t)m_pad * s_pad * sizeof(T) * 3));
  T* Od = (T*)tmp; T* Zd = Od + m_pad * s_pad; T* Zb = Zd + m_pad * s_pad;
  CK(sc.alloc(&tmp, (size_t)m_pad * sizeof(double)));
  double* rs = (double*)tmp;
  CK(cudaMemsetAsync(Od, 0, (size_t)m_pad * s_pad * sizeof(T) * 2, s));  // zero padding rows / columns of Obar and Z
  CK(cudaMemcpy2DAsync(Od, (size_t)m_pad * sizeof(T), out_bar, (size_t)M * sizeof(T), (size_t)M * sizeof(T), (size_t)S, kin, s));
  CK(cudaMemcpy2DAsync(Zd, (size_t)m_pad * sizeof(T), Z, (size_t)M * sizeof(T), (size_t)M * sizeof(T), (size_t)S, kin, s));
  sample_pullback<T>(ctx, (const T*)Lf, ldf, Vs, M, m_pad, S, s_pad, Od, Zd, Zb, rs, Lt, Ws, false);
  if (std::is_same<T, double>::value)
    CK(cudaMemcpyAsync(mubar, rs, (size_t)M * sizeof(double), cudaMemcpyDeviceToDevice, s));
  else
    launch_cast<double, float>(rs, (float*)mubar, M, s);
  if (z_bar_out)
    CK(cudaMemcpy2DAsync(z_bar_out, (size_t)M * sizeof(T), Zb, (size_t)m_pad * sizeof(T), (size_t)M * sizeof(T), (size_t)S, kout, s));
  rc = download<T>(ctx, mean_s_diag_out, mubar, (size_t)M, false);
  if (rc) return rc;
  drop(Od); drop(Lt); drop(Lf); drop(Dinv);
  if (Vs) drop(Vs);

  // ---- training side: P = L^-T A with room for alpha (post_pred_tail), then the blocks and the reductions
  if (want_beta) {
    CK(sc.alloc(&tmp, (size_t)n_pad * (m_pad + XK) * sizeof(T)));
    T* P = (T*)tmp;
    CK(cudaMemcpyAsync(P, A, (size_t)n_pad * m_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
    drop(A);
    backward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, P, n_pad, m_pad);
    rc = post_pred_tail<T>(p, sc, layout, Xst, M, Ws, P, want_red, grad_out, noise_diag_out, mean_diag_out, y_bar_out,
                           x_grad_out, noise_s_diag_out, xs_grad_out);
    if (rc) return rc;
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

// ---- pullback of mean_and_var(posterior(fx, y)(x*)) on a handle from agp_fit (agp.h agp_post_mean_var_grad).  With
// A = L^-1 K_xs and P = C^-1 K_xs = L^-T A (forward_subst_multi, then backward_subst_multi: N^2 M, no L^-1 or C^-1), the
// cotangents mbar of the means and vbar of the variances are the held-out gradient's mubar and Sigmabar = diag(vbar):
//   Kbar_sx[j, n] = mbar_j alpha_n - 2 vbar_j P[n, j],  beta = P mbar,  Cbar = P diag(vbar) P' - 1/2 (beta alpha' + alpha beta').
// mu*, Sigma and its factor never enter: the call takes neither the test mean nor the test noise.
//   - x* side: xs_grad_out always comes from launch_cross_grad_x, one pass over the N x M pairs with Kbar_sx formed from P
//     on the fly (post_xs_grad.cu), whatever else is asked for.
//   - training side: the kernel, noise and x outputs run post_pred_tail unchanged with Ws = -2 diag(vbar) and mubar = mbar
//     (its test-side outputs NULL); y_bar_out and mean_diag_out alone need only beta, one GEMV, and skip the stacked pass.
// Without a kernel, noise or x output the call allocates A and P (P = A in place: about NM elements) and the cross
// pass's O((N + M) D); the training side adds the tail's m_pad (m_pad + 16) Ws and (N + M)^2 stacked W.
template <typename T>
int post_mean_var_grad_impl(agp_post* p, int layout, const void* Xs, int64_t M, const void* mean_bar, const void* var_bar,
                            double* grad_out, void* noise_diag_out, void* mean_diag_out, void* y_bar_out, void* x_grad_out,
                            void* xs_grad_out) {
  agp_ctx* ctx = p->ctx;
  if (!Xs) { ctx->err = "Xs is NULL"; return AGP_ERR_INVALID; }
  if (M <= 0) { ctx->err = "M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  int rc = logpdf_grad_prelude<T>(p, layout);
  if (rc) return rc;
  cudaStream_t s = ctx->stream;
  const int64_t N = p->n, n_pad = p->n_pad, m_pad = round_up(M, TILE);
  const int D = p->D;
  constexpr int64_t XK = POST_XK;
  const bool want_red = grad_out || noise_diag_out || x_grad_out;
  const bool want_beta = want_red || mean_diag_out || y_bar_out;
  if (!want_beta && !xs_grad_out) return AGP_OK;
  Scratch sc(ctx);
  void* tmp = nullptr;
  auto drop = [&](void* q) { sc.release(q); cudaFreeAsync(q, s); };

  // the cotangents on the device, m_pad values each with zero padding (NULL: zeros)
  CK(sc.alloc(&tmp, (size_t)m_pad * 2 * sizeof(T)));
  T* mbar = (T*)tmp;
  T* vbar = mbar + m_pad;
  CK(cudaMemsetAsync(mbar, 0, (size_t)m_pad * 2 * sizeof(T), s));
  const cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (mean_bar) CK(cudaMemcpyAsync(mbar, mean_bar, (size_t)M * sizeof(T), kin, s));
  if (var_bar) CK(cudaMemcpyAsync(vbar, var_bar, (size_t)M * sizeof(T), kin, s));

  // ---- forward: A = L^-1 K_xs, then P = L^-T A (with room for the tail's alpha column when the tail runs)
  T *Xst = nullptr, *A = nullptr;
  rc = post_cross<T>(p, sc, layout, Xs, M, m_pad, &Xst, &A);
  if (rc) return rc;
  forward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, A, n_pad, m_pad);
  T* P = A;
  if (want_red) {
    CK(sc.alloc(&tmp, (size_t)n_pad * (m_pad + XK) * sizeof(T)));
    P = (T*)tmp;
    CK(cudaMemcpyAsync(P, A, (size_t)n_pad * m_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
    drop(A);
  }
  backward_subst_multi<T>(ctx, (const T*)p->L, p->lda, (const T*)p->Dinv, n_pad, P, n_pad, m_pad);

  // ---- x* side: one pass over the N x M pairs
  if (xs_grad_out) {
    const CompositeDesc one = single_kernel_desc(p->k.family, p->k.variance, p->k.linear_c);
    const CompositeDesc* cd = &one;
    double mult = 1.0;
    const T* ard = nullptr;
    if (p->comp) {
      cd = &p->comp->desc;
    } else {
      if (p->k.transform == AGP_T_SCALE) mult = p->k.scale;
      else if (p->k.transform == AGP_T_ARD) ard = (const T*)p->ard;
    }
    CK(sc.alloc(&tmp, (size_t)cross_grad_x_part_len(M, N, D, cd->nacc) * sizeof(double)));
    double* part = (double*)tmp;
    CK(sc.alloc(&tmp, (size_t)M * D * sizeof(T)));
    T* xsg = (T*)tmp;
    launch_cross_grad_x<T>(Xst, M, (const T*)p->Xt, N, D, P, n_pad, (const T*)p->alpha, mbar, vbar, *cd, mult, ard, layout,
                           part, xsg, s);
    rc = download<T>(ctx, xs_grad_out, xsg, (size_t)M * D, false);
    if (rc) return rc;
  }

  // ---- training side
  if (want_red) {  // Ws = -2 diag(vbar) and mubar = mbar in column m_pad, then post_pred_tail
    CK(sc.alloc(&tmp, (size_t)m_pad * (m_pad + XK) * sizeof(T)));
    T* Ws = (T*)tmp;
    CK(cudaMemsetAsync(Ws, 0, (size_t)m_pad * (m_pad + XK) * sizeof(T), s));
    CK(cudaMemcpy2DAsync(Ws, (size_t)(m_pad + 1) * sizeof(T), vbar, sizeof(T), sizeof(T), (size_t)M,
                         cudaMemcpyDeviceToDevice, s));  // the diagonal
    launch_scale<T>(Ws, m_pad * m_pad, -2.0, s);
    CK(cudaMemcpyAsync(Ws + m_pad * m_pad, mbar, (size_t)M * sizeof(T), cudaMemcpyDeviceToDevice, s));
    rc = post_pred_tail<T>(p, sc, layout, Xst, M, Ws, P, true, grad_out, noise_diag_out, mean_diag_out, y_bar_out,
                           x_grad_out, nullptr, nullptr);
    if (rc) return rc;
  } else if (want_beta) {  // ybar = beta = P mbar, mbar at x = -beta (the tail's GEMV)
    CK(sc.alloc(&tmp, (size_t)n_pad * 2 * sizeof(T)));
    T* beta = (T*)tmp;
    T* nbeta = beta + n_pad;
    CK(cudaMemsetAsync(beta, 0, (size_t)n_pad * 2 * sizeof(T), s));
    launch_gemv_n_acc<T>(P, n_pad, N, M, mbar, beta, s);
    rc = download<T>(ctx, y_bar_out, beta, (size_t)N, false);
    if (rc) return rc;
    if (mean_diag_out) {
      CK(cudaMemcpyAsync(nbeta, beta, (size_t)n_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
      launch_scale<T>(nbeta, n_pad, -1.0, s);
      rc = download<T>(ctx, mean_diag_out, nbeta, (size_t)N, false);
      if (rc) return rc;
    }
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

template <typename T>
int gram_impl(agp_ctx* ctx, const agp_kernel* k, int layout, const void* X, int64_t N, int D, const void* Z,
              int64_t M, const agp_noise* noise, void* K_out) {
  int rc = check_kernel(ctx, k, D);
  if (rc) return rc;
  if (N <= 0 || (Z && M <= 0)) { ctx->err = "empty input"; return AGP_ERR_DIM_MISMATCH; }
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  CompState comp_local, *comp = nullptr;
  if (k->family == AGP_COMPOSITE) { rc = comp_build<T>(ctx, k, D, &comp_local); if (rc) return rc; comp = &comp_local; }
  Scratch sc(ctx);
  const int64_t n_pad = round_up(N, 64);
  const int64_t cols = Z ? M : N, c_pad = round_up(cols, 64);
  T *ard_d = nullptr, *noise_d = nullptr, *Xt = nullptr, *Zt = nullptr;
  if (k->transform == AGP_T_ARD) { rc = upload<T>(ctx, sc, k->ard, D, true, &ard_d); if (rc) return rc; }
  if (noise && noise->kind == 1) { rc = upload<T>(ctx, sc, noise->v, N, true, &noise_d); if (rc) return rc; }
  rc = prep_points<T>(ctx, sc, k, ard_d, layout, X, N, n_pad, D, &Xt, false);
  if (rc) return rc;
  if (Z) { rc = prep_points<T>(ctx, sc, k, ard_d, layout, Z, M, c_pad, D, &Zt, false); if (rc) return rc; }
  if (comp) { rc = comp_upload<T>(ctx, sc, comp, false); if (rc) return rc; }
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)n_pad * c_pad * sizeof(T)));
  GramParams gp{};
  fill_gram_params<T>(gp, k, Z ? 0 : 1, 0, N, cols, Z ? nullptr : noise, noise_d, comp);
  launch_gram<T>(Xt, Z ? Zt : Xt, n_pad, c_pad, D, (T*)tmp, n_pad, gp, s);
  cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  CK(cudaMemcpy2DAsync(K_out, (size_t)N * sizeof(T), tmp, (size_t)n_pad * sizeof(T), (size_t)N * sizeof(T), (size_t)cols, kout, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}




// ---- VFE (Titsias) : elbo / dtc / approximate posterior --------------------------------------------
// Follows /root/reference/src/sparse_approximations.jl:289-305 (_compute_intermediates), :248-254 (elbo),
// :58-75 (posterior), but STREAMS the data dimension: K_zx is generated chunk by chunk, scaled by
// Sigma_y^-1/2, solved against chol(K_zz) and folded into D = A A' (M x M), b = A delta and ||A||_F^2,
// so the M x N matrix A (32.8 GB at config C5) never exists.
//
// What the gradient (vfe_grad_impl) needs from the pass: the factors, m_e, D = Lam - I, the prepared points and the
// per-point vectors.  `after` runs while they are alive; without it the pass launches exactly what the objectives need.
template <typename T>
struct VfePass {
  int64_t N, M, m_pad, lda, cap;
  int D;
  const T *Lz, *Dz, *Lm, *Dl, *me, *Dcopy, *Zt, *Xt, *kd, *delta, *isn, *noise_v, *ard;
  T* B;  // pass 1's chunk buffer (m_pad x cap), free for reuse
  double noise_s, elbo, dtc;
};
template <typename T> using VfeAfter = std::function<int(const VfePass<T>&)>;

template <typename T>
int vfe_core(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout,
             const void* X, int64_t N, int D, const void* Zind, int64_t M, const agp_noise* jitter, const void* y,
             void* elbo_out, void* dtc_out, agp_vfe_post** post_out, const VfeAfter<T>* after = nullptr) {
  if (k && k->family == AGP_COMPOSITE) {
    ctx->err = "composite kernels are supported on the exact path only (not VFE)";
    return AGP_ERR_UNSUPPORTED;
  }
  int rc = check_kernel(ctx, k, D);
  if (rc) return rc;
  if (N <= 0 || M <= 0) { ctx->err = "N and M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (!X || !Zind || !y) { ctx->err = "X/Z/y is NULL"; return AGP_ERR_INVALID; }
  static const agp_mean zero_mean{0, 0.0, nullptr};
  static const agp_noise default_noise{0, 1e-18, nullptr};
  if (!mean) mean = &zero_mean;
  if (!noise) noise = &default_noise;
  if (!jitter) jitter = &default_noise;
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  Scratch sc(ctx);
  const bool keep = post_out != nullptr;
  // + TILE: a rank's shard start is not tile-aligned, and the chunk Gram reads whole 128-point slabs from it
  const int64_t m_pad = round_up(M, TILE), lda = m_pad + TILE, n_padN = round_up(N, TILE) + TILE;
  const int nblk = (int)(m_pad / TILE);
  CK(cudaEventRecord(ctx->ev[0], s));
  T *ard_d = nullptr, *mean_d = nullptr, *noise_d = nullptr, *jit_d = nullptr, *yd = nullptr, *Zt = nullptr, *Xt = nullptr;
  if (k->transform == AGP_T_ARD) { rc = upload<T>(ctx, sc, k->ard, D, true, &ard_d); if (rc) return rc; }
  if (mean->kind == 2) { rc = upload<T>(ctx, sc, mean->v, N, true, &mean_d); if (rc) return rc; }
  if (noise->kind == 1) { rc = upload<T>(ctx, sc, noise->v, N, true, &noise_d); if (rc) return rc; }
  if (jitter->kind == 1) { rc = upload<T>(ctx, sc, jitter->v, M, true, &jit_d); if (rc) return rc; }
  rc = upload<T>(ctx, sc, y, N, false, &yd); if (rc) return rc;
  rc = prep_points<T>(ctx, sc, k, ard_d, layout, Zind, M, m_pad, D, &Zt, keep); if (rc) return rc;
  rc = prep_points<T>(ctx, sc, k, ard_d, layout, X, N, n_padN, D, &Xt, false); if (rc) return rc;
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)n_padN * 3 * sizeof(T)));
  T* kd = (T*)tmp; T* delta = kd + n_padN; T* isn = delta + n_padN;
  CK(cudaMemsetAsync(kd, 0, (size_t)n_padN * 3 * sizeof(T), s));
  CK(sc.alloc(&tmp, (size_t)(2 * nblk + TILE + 16) * sizeof(double)));
  double* dscal = (double*)tmp;  // [0..3] prep scalars + ||A||^2, [8..8+nblk) logdet Kzz, [8+nblk..) logdet Lam, then sq
  CK(cudaMemsetAsync(dscal, 0, (size_t)(2 * nblk + TILE + 16) * sizeof(double), s));
  double* ld_z = dscal + 8; double* ld_l = ld_z + nblk; double* sq = ld_l + nblk;
  CK(sc.alloc(&tmp, sizeof(int)));
  int* dinfo = (int*)tmp;
  CK(cudaMemsetAsync(dinfo, 0, sizeof(int), s));
  // data shard of this rank (multi-GPU: the N dimension is partitioned, ONE all-reduce at the end -- SURVEY s8e)
  int64_t n_lo = 0, n_hi = N;
  if (ctx->nccl) {
    const int64_t per = (N + ctx->nranks - 1) / ctx->nranks;
    n_lo = (int64_t)ctx->rank * per; if (n_lo > N) n_lo = N;
    n_hi = n_lo + per; if (n_hi > N) n_hi = N;
  }
  launch_kdiag<T>(Xt, N, D, k->family, k->variance, k->linear_c, kd, s);
  launch_vfe_prep<T>(yd + n_lo, n_hi - n_lo, mean->kind, mean->c, mean_d ? mean_d + n_lo : nullptr, noise->kind, noise->s,
                     noise_d ? noise_d + n_lo : nullptr, kd + n_lo, delta + n_lo, isn + n_lo, dscal, s);

  // factor buffers
  void *Lzv = nullptr, *Dzv = nullptr, *Lmv = nullptr, *Dlv = nullptr, *mev = nullptr;
  CK(cudaMallocAsync(&Lzv, (size_t)lda * m_pad * sizeof(T), s));
  CK(cudaMallocAsync(&Dzv, (size_t)nblk * TILE * TILE * sizeof(T), s));
  CK(cudaMallocAsync(&Lmv, (size_t)lda * m_pad * sizeof(T), s));
  CK(cudaMallocAsync(&Dlv, (size_t)nblk * TILE * TILE * sizeof(T), s));
  CK(cudaMallocAsync(&mev, (size_t)m_pad * 2 * sizeof(T), s));
  if (!keep) { sc.ptrs.push_back(Lzv); sc.ptrs.push_back(Dzv); sc.ptrs.push_back(Lmv); sc.ptrs.push_back(Dlv); sc.ptrs.push_back(mev); }
  T* Lz = (T*)Lzv; T* Dz = (T*)Dzv; T* Lm = (T*)Lmv; T* Dl = (T*)Dlv; T* bvec = (T*)mev; T* rwork = bvec + m_pad;
  agp_vfe_post* vp = nullptr;
  if (keep) {
    vp = new agp_vfe_post();
    vp->ctx = ctx; vp->dtype = sizeof(T) == 8 ? AGP_F64 : AGP_F32; vp->m = M; vp->m_pad = m_pad; vp->lda = lda; vp->D = D;
    vp->U = Lzv; vp->Udinv = Dzv; vp->Lam = Lmv; vp->Ldinv = Dlv; vp->Zt = Zt; vp->m_e = mev;
    vp->k = *k; vp->k.ard = nullptr;
    if (ard_d) { sc.release(ard_d); vp->ard = ard_d; }
    vp->mean_kind = mean->kind == 2 ? 0 : mean->kind; vp->mean_c = mean->c;
  }
  // every early return (CK / CKN failures, non-PD) releases the half-built handle and its buffers
  struct VfeGuard { agp_vfe_post* p; ~VfeGuard() { if (p) agp_vfe_post_free(p); } } vguard{vp};
  auto fail = [&](int code) { return code; };

  // (1) chol(K_zz + jitter)
  GramParams gz{};
  fill_gram_params<T>(gz, k, 1, 1, M, M, jitter, jit_d);
  launch_gram<T>(Zt, Zt, m_pad, m_pad, D, Lz, lda, gz, s);
  launch_border_init<T>(Lz, lda, m_pad, m_pad, (const T*)nullptr, m_pad, 0, 0, 0.0, (const T*)nullptr, s);
  prof_begin(ctx);
  cholesky_inplace<T>(ctx, Lz, lda, m_pad, lda, Dz, ld_z, dinfo);
  CK(cudaEventRecord(ctx->ev[1], s));

  // (2) stream the data: D += A_c A_c', b += A_c delta_c, ||A||_F^2
  CK(cudaMemsetAsync(Lm, 0, (size_t)lda * m_pad * sizeof(T), s));
  CK(cudaMemsetAsync(bvec, 0, (size_t)m_pad * 2 * sizeof(T), s));
  int64_t cap = (int64_t)(2.0e9 / ((double)m_pad * sizeof(T)));
  { const int64_t c_env = env_int64("AGP_VFE_CHUNK", 0); if (c_env > 0) cap = c_env; }  // tests: force small chunks
  cap = cap / TILE * TILE;
  if (cap < TILE) cap = TILE;
  if (cap > n_padN) cap = n_padN;
  // D += A_c A_c' on the tensor cores: the chunk is ONE long-K product (K = chunk width); the int32 accumulators of the
  // sliced kernel hold (d+1) * K * 64^2 < 2^31, so K <= 32768 keeps every slice count exact
  const bool syrk_tc = resolve_tensor_mode<T>(ctx, (int64_t)1 << 20) == 1 && m_pad >= 1024;
  if (syrk_tc && cap > 32768) cap = 32768;
  constexpr int is_f32 = std::is_same<T, double>::value ? 0 : 1;
  void* Bv = nullptr;
  CK(sc.alloc(&Bv, (size_t)m_pad * cap * sizeof(T)));
  T* B = (T*)Bv;
  for (int64_t c0 = n_lo; c0 < n_hi; c0 += cap) {
    const int64_t nc = (n_hi - c0 < cap) ? (n_hi - c0) : cap;
    const int64_t nc_pad = round_up(nc, TILE);
    GramParams gx{};
    fill_gram_params<T>(gx, k, 0, 0, M, nc, nullptr, nullptr);
    launch_gram<T>(Zt, Xt + c0 * D, m_pad, nc_pad, D, B, m_pad, gx, s);
    launch_scale_cols<T>(B, m_pad, m_pad, nc, isn + c0, s);
    forward_subst_multi<T>(ctx, Lz, lda, Dz, m_pad, B, m_pad, nc_pad);
    bool acc_done = false;
    if (syrk_tc && nc_pad >= 1024 && ensure_oz2<T>(ctx, m_pad, (int)nc_pad, false, s) && ctx->oz2.bulk == 2) {
      ozaki_prepare_ex(ctx->oz2, B, is_f32, 0, m_pad, m_pad, 0, s);
      acc_done = ozaki_update_ex(ctx->oz2, Lm, is_f32, lda, m_pad, m_pad, 0, 1.0, 0, 0, 0, 0, s) == 0;
    }
    if (!acc_done) {
      GemmArgs g{};
      g.A = B; g.lda = m_pad; g.B = B; g.ldb = m_pad; g.C = Lm; g.ldc = lda;
      g.M = m_pad; g.N = m_pad; g.K = nc_pad; g.beta_one = 1; g.lower_only = 1;
      launch_gemm<T>(g, s);
    }
    launch_gemv_n_acc<T>(B, m_pad, m_pad, nc, delta + c0, bvec, s);
    launch_sumsq<T>(B, m_pad * nc_pad, dscal + 3, s);
  }
  if (ctx->nccl) {  // the one exchange step: D (M x M), b (M) and the three scalars
    CKN(ncclAllReduce(Lm, Lm, (size_t)lda * m_pad, NcclType<T>::v, ncclSum, ctx->nccl, s));
    CKN(ncclAllReduce(bvec, bvec, (size_t)m_pad, NcclType<T>::v, ncclSum, ctx->nccl, s));
    CKN(ncclAllReduce(dscal, dscal, 4, ncclDouble, ncclSum, ctx->nccl, s));
  }
  CK(cudaEventRecord(ctx->ev[2], s));

  // (3) Lambda = chol(D + I), with b riding in the border row
  T* Dcopy = nullptr;
  if (after) {
    CK(sc.alloc(&tmp, (size_t)lda * m_pad * sizeof(T)));
    Dcopy = (T*)tmp;
    CK(cudaMemcpyAsync(Dcopy, Lm, (size_t)lda * m_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
  }
  launch_add_diag<T>(Lm, lda, m_pad, 1.0, s);
  launch_border_init<T>(Lm, lda, m_pad, m_pad, bvec, m_pad, 1, 0, 0.0, (const T*)nullptr, s);
  cholesky_inplace<T>(ctx, Lm, lda, m_pad, lda, Dl, ld_l, dinfo);
  launch_extract_v<T>(Lm, lda, m_pad, 1, rwork, sq, s);
  if (keep || after) {
    CK(sc.alloc(&tmp, (size_t)(nblk + 1) * sizeof(int)));
    int* dflags = (int*)tmp;
    launch_bwd_solve<T>(Lm, lda, Dl, nblk, rwork, dflags, s);       // m_e = Lambda^-1 b
    CK(cudaMemcpyAsync(bvec, rwork, (size_t)m_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));  // m_e kept in slot 0
  }
  CK(cudaEventRecord(ctx->ev[3], s));
  std::vector<double> h((size_t)(2 * nblk + 16 + 1));
  int h_info = 0;
  CK(cudaMemcpyAsync(h.data(), dscal, (size_t)(2 * nblk + 16 + 1) * sizeof(double), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&h_info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]); ctx->timings[0] = ms;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]); ctx->timings[3] = ms;
  cudaEventElapsedTime(&ms, ctx->ev[1], ctx->ev[2]); ctx->timings[6] = ms;
  ctx->timings[7] = ctx->profile ? prof_total_ms(ctx) : 0.0;
  if (h_info != 0) {
    ctx->info = h_info;
    ctx->err = "VFE: K_zz + jitter or A A' + I is not positive definite";
    return fail(AGP_ERR_NOT_POSDEF);
  }
  double logdet_lam = 0.0;
  for (int b = 0; b < nblk; ++b) logdet_lam += h[8 + nblk + b];
  logdet_lam *= 2.0;
  const double log2pi = 1.8378770664093454835606594728112;
  const double sqv = h[8 + 2 * nblk];
  const double dtc = -0.5 * ((double)N * log2pi + h[0] + logdet_lam + h[1] - sqv);
  const double elbo = dtc - 0.5 * (h[2] - h[3]);
  T e = (T)elbo, dd = (T)dtc;
  if (elbo_out) memcpy(elbo_out, &e, sizeof(T));
  if (dtc_out) memcpy(dtc_out, &dd, sizeof(T));
  if (after) {
    const VfePass<T> st{N, M, m_pad, lda, cap, D, Lz, Dz, Lm, Dl, bvec, Dcopy, Zt, Xt, kd, delta, isn, noise_d, ard_d,
                        B, noise->s, elbo, dtc};
    rc = (*after)(st);
    if (rc) return fail(rc);
  }
  vguard.p = nullptr;
  if (keep) *post_out = vp;
  return AGP_OK;
}

// ---- gradient of the VFE objectives (agp_vfe_elbo_grad; the formulas are in agp.h and vfe_grad.cu) ----------------
int vfe_grad_check(agp_ctx* ctx, const agp_kernel* k, int layout, int objective) {
  if (objective != 0 && objective != 1) { ctx->err = "objective must be 0 (elbo) or 1 (DTC)"; return AGP_ERR_INVALID; }
  int rc = check_layout(ctx, layout);
  if (rc) return rc;
  if (k && k->family == AGP_COMPOSITE) { ctx->err = "composite kernels are supported on the exact path only (not VFE)"; return AGP_ERR_UNSUPPORTED; }
  if (ctx->nccl) { ctx->err = "the VFE gradient runs on a single-GPU context"; return AGP_ERR_UNSUPPORTED; }
  return AGP_OK;
}


// Pass 1 is vfe_core's.  Then, once: V_z = L_z^-1 and V_m = L_m^-1 by the forward substitution on the identity,
// Lam^-1 = V_m' V_m, H and E, R = V_z' H V_z, P = V_z' E V_z = -2 Kbar_zz and r = V_z' m_e (O(M^3), tile GEMMs).  The K_zz
// part goes through the exact path's reductions with alpha = 0 and C^-1 = P: grad_reduce_kernel gives
// 1/2 sum (-P) o dK_zz = sum Kbar_zz o dK_zz, grad_x_kernel gives sum_m' (-P) d1k = 2 sum Kbar_zz d1k.  Pass 2 streams the
// data in pass 1's chunks: K_zx,c by the Gram kernel, G = R K_zx,c by the tile GEMM, then vfe_cross_grad_kernel and
// vfe_point_grad_kernel, and with x_grad_out vfe_x_grad_kernel and vfe_x_finish_kernel on the same G (vfe_grad_x.cu).
template <typename T>
int vfe_grad_impl(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout,
                  const void* X, int64_t N, int D, const void* Zind, int64_t M, const agp_noise* jitter, const void* y,
                  int objective, void* value_out, double* grad_out, void* noise_diag_out, void* mean_diag_out,
                  void* z_grad_out, void* x_grad_out) {
  const double c = objective == 0 ? 1.0 : 0.0;
  const VfeAfter<T> grad = [&](const VfePass<T>& p) -> int {
    cudaStream_t s = ctx->stream;
    const int64_t mp = p.m_pad, mm = mp * mp;
    const bool linear = k->family == AGP_LINEAR;
    const int want_ard = k->transform == AGP_T_ARD ? 1 : 0;
    Scratch sc(ctx);
    void* tmp = nullptr;
    CK(sc.alloc(&tmp, (size_t)(mm * 6 + mp * 2) * sizeof(T)));
    T* Vz = (T*)tmp; T* W1 = Vz + mm; T* Li = W1 + mm; T* H = Li + mm; T* E = H + mm; T* R = E + mm;
    T* rv = R + mm; T* az = rv + mp;
    T* P = H;  // V_z' E V_z takes H's place once R is formed
    auto gemm = [&](const T* A, int ak, const T* B, int bk, T* C) {
      GemmArgs g{};
      g.A = A; g.lda = mp; g.a_kmajor = ak;
      g.B = B; g.ldb = mp; g.b_kmajor = bk;
      g.C = C; g.ldc = mp; g.M = mp; g.N = mp; g.K = mp;
      launch_gemm<T>(g, s);
    };
    CK(cudaMemsetAsync(Vz, 0, (size_t)mm * 2 * sizeof(T), s));
    CK(cudaMemsetAsync(az, 0, (size_t)mp * sizeof(T), s));
    launch_add_diag<T>(Vz, mp, mp, 1.0, s);
    launch_add_diag<T>(W1, mp, mp, 1.0, s);
    forward_subst_multi<T>(ctx, p.Lz, p.lda, p.Dz, mp, Vz, mp, mp);  // V_z
    forward_subst_multi<T>(ctx, p.Lm, p.lda, p.Dl, mp, W1, mp, mp);  // V_m
    gemm(W1, 1, W1, 1, Li);                                           // Lam^-1 = V_m' V_m
    launch_vfe_hz<T>(Li, p.Dcopy, p.lda, p.me, M, mp, c, H, E, s);
    gemm(H, 0, Vz, 1, W1);
    gemm(Vz, 1, W1, 1, R);                                            // R = V_z' H V_z
    gemm(E, 0, Vz, 1, W1);
    gemm(Vz, 1, W1, 1, P);                                            // P = V_z' E V_z
    launch_gemv_t<T>(Vz, mp, mp, mp, p.me, 0, 0.0, (const T*)nullptr, rv, s);  // r = V_z' m_e

    const int nsums = 5 + D;
    CK(sc.alloc(&tmp, (size_t)(nsums + 2) * sizeof(double)));
    double* sums = (double*)tmp;
    double* nm = sums + nsums;
    CK(cudaMemsetAsync(sums, 0, (size_t)(nsums + 2) * sizeof(double), s));
    launch_grad_reduce<T>(p.Zt, D, M, mp, P, mp, az, k->family, k->linear_c, want_ard, sums, (T*)nullptr, s);
    const double mult = k->transform == AGP_T_SCALE ? k->scale : 1.0;
    const T* ard = want_ard ? p.ard : nullptr;
    T *zz = nullptr, *zout = nullptr;
    if (z_grad_out) {  // K_zz part of the inducing-point gradient, in the caller's layout
      const CompositeDesc one = single_kernel_desc(k->family, k->variance, k->linear_c);
      CK(sc.alloc(&tmp, (size_t)grad_x_part_len(M, D, 1) * sizeof(double)));
      double* part = (double*)tmp;
      CK(sc.alloc(&tmp, (size_t)M * D * 2 * sizeof(T)));
      zz = (T*)tmp; zout = zz + M * D;
      launch_grad_x<T>(p.Zt, D, M, P, mp, az, one, mult, ard, layout, part, zz, s);
    }

    // pass 2
    const int64_t cap = p.cap;
    int nrb = 0, nsplit = 0;
    vfe_cross_shape(mp, cap, &nrb, &nsplit);
    CK(sc.alloc(&tmp, (size_t)mp * cap * sizeof(T)));
    T* Bk = p.B; T* G = (T*)tmp;
    // G on the int8-slice general product wherever pass 1 runs its long-K product on the tensor cores (the same rule):
    // R is sliced once into rows [0, m_pad) of the workspace, each chunk of K_zx behind it
    constexpr int is_f32 = std::is_same<T, double>::value ? 0 : 1;
    bool g_tc = resolve_tensor_mode<T>(ctx, (int64_t)1 << 20) == 1 && mp >= 1024 && mp <= 32768 &&
                ensure_oz2<T>(ctx, mp + cap, (int)mp, false, s) && ctx->oz2.bulk == 2;
    if (g_tc) ozaki_prepare_ex(ctx->oz2, R, is_f32, 0, mp, mp, 0, s);
    CK(sc.alloc(&tmp, (size_t)(2 * nrb * cap + (int64_t)nsplit * D * mp) * sizeof(double)));
    double* qpart = (double*)tmp; double* upart = qpart + nrb * cap; double* zpart = upart + nrb * cap;
    CK(cudaMemsetAsync(zpart, 0, (size_t)nsplit * D * mp * sizeof(double), s));
    T *nd = nullptr, *md = nullptr;
    if (noise_diag_out) { CK(sc.alloc(&tmp, (size_t)N * sizeof(T))); nd = (T*)tmp; }
    if (mean_diag_out) { CK(sc.alloc(&tmp, (size_t)N * sizeof(T))); md = (T*)tmp; }
    // the input gradient: per-chunk partials (row ranges x (D + 1) x cap), written in place under AGP_MEM_DEVICE
    int xsplit = 0;
    double* xpart = nullptr;
    T* xout = nullptr;
    const bool x_dev = ctx->memspace == AGP_MEM_DEVICE || ctx->out_dev_override;
    if (x_grad_out) {
      vfe_x_shape(mp, cap, &xsplit);
      CK(sc.alloc(&tmp, (size_t)xsplit * (D + 1) * cap * sizeof(double)));
      xpart = (double*)tmp;
      if (x_dev) xout = (T*)x_grad_out;
      else { CK(sc.alloc(&tmp, (size_t)N * D * sizeof(T))); xout = (T*)tmp; }
    }
    for (int64_t c0 = 0; c0 < N; c0 += cap) {
      const int64_t nc = (N - c0 < cap) ? (N - c0) : cap;
      const int64_t nc_pad = round_up(nc, TILE);
      GramParams gx{};
      fill_gram_params<T>(gx, k, 0, 0, M, nc, nullptr, nullptr);
      launch_gram<T>(p.Zt, p.Xt + c0 * D, mp, nc_pad, D, Bk, mp, gx, s);
      bool done = false;
      if (g_tc) {  // G = R K_zx,c
        CK(cudaMemsetAsync(G, 0, (size_t)mp * nc_pad * sizeof(T), s));
        ozaki_prepare_ex(ctx->oz2, Bk, is_f32, 1, mp, nc_pad, mp, s);
        done = ozaki_update_ex(ctx->oz2, G, is_f32, mp, mp, nc_pad, 1, 1.0, 0, 0, mp, 0, s) == 0;
      }
      if (!done) {
        GemmArgs g{};
        g.A = R; g.lda = mp; g.a_kmajor = 0;
        g.B = Bk; g.ldb = mp; g.b_kmajor = 1;
        g.C = G; g.ldc = mp; g.M = mp; g.N = nc_pad; g.K = mp;
        launch_gemm<T>(g, s);
      }
      launch_vfe_cross_grad<T>(p.Zt, M, mp, p.Xt + c0 * D, nc, D, G, mp, rv, p.delta + c0, p.isn + c0, k->family, k->variance,
                               k->linear_c, want_ard, nsplit, sums, qpart, upart, cap, zpart, s);
      launch_vfe_point_grad<T>(qpart, upart, cap, nrb, nc, p.delta + c0, p.isn + c0, p.kd + c0, p.noise_v ? 1 : 0, p.noise_s,
                               p.noise_v ? p.noise_v + c0 : nullptr, c, p.Xt + c0 * D, D, linear ? 1 : 0, k->linear_c,
                               want_ard, sums, nm, nd ? nd + c0 : nullptr, md ? md + c0 : nullptr, s);
      if (x_grad_out) {
        launch_vfe_x_grad<T>(p.Zt, M, mp, p.Xt + c0 * D, nc, D, G, mp, rv, p.delta + c0, p.isn + c0, k->family, xsplit, xpart,
                             cap, s);
        launch_vfe_x_finish<T>(xpart, xsplit, cap, nc, D, p.Xt + c0 * D, p.isn + c0, linear ? 1 : 0, k->variance, c, mult,
                               ard, layout, N, c0, xout, s);
      }
    }
    if (x_grad_out && !x_dev) { int rc = download<T>(ctx, x_grad_out, xout, (size_t)N * D, false); if (rc) return rc; }
    if (z_grad_out) {
      launch_vfe_z_finish<T>(zpart, nsplit, mp, M, D, mult * k->variance, ard, layout, zz, zout, s);
      int rc = download<T>(ctx, z_grad_out, zout, (size_t)M * D, false); if (rc) return rc;
    }
    { int rc = download<T>(ctx, noise_diag_out, nd, (size_t)N, false); if (rc) return rc; }
    { int rc = download<T>(ctx, mean_diag_out, md, (size_t)N, false); if (rc) return rc; }
    std::vector<double> h((size_t)nsums + 2);
    std::vector<T> ard_h((size_t)(D > 0 ? D : 1));
    CK(cudaMemcpyAsync(h.data(), sums, h.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (want_ard) CK(cudaMemcpyAsync(ard_h.data(), p.ard, (size_t)D * sizeof(T), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    if (value_out) { const T v = (T)(objective == 0 ? p.elbo : p.dtc); memcpy(value_out, &v, sizeof(T)); }
    if (!grad_out) return AGP_OK;
    single_kernel_grad<T>(*k, D, h.data(), ard_h.data(), grad_out);
    grad_out[3] = h[(size_t)nsums];
    grad_out[4] = h[(size_t)nsums + 1];
    return AGP_OK;
  };
  return vfe_core<T>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, nullptr, nullptr, nullptr, &grad);
}

// fp32 problems: the value is the fp32 pass's, the value agp_vfe_elbo returns; the gradient is formed in fp64 on the
// same problem converted to fp64 (pass 1 included), because its adjoints are differences of terms up to ~1e5 times larger
// than the result (agp.h).  Inputs and outputs keep the caller's memory space.
int vfe_grad_f32(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout, const void* X,
                 int64_t N, int D, const void* Zind, int64_t M, const agp_noise* jitter, const void* y, int objective,
                 void* value_out, double* grad_out, void* noise_diag_out, void* mean_diag_out, void* z_grad_out,
                 void* x_grad_out) {
  int rc = check_kernel(ctx, k, D);
  if (rc) return rc;
  if (N <= 0 || M <= 0) { ctx->err = "N and M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (!X || !Zind || !y) { ctx->err = "X/Z/y is NULL"; return AGP_ERR_INVALID; }
  if (value_out) {
    float v[2];
    rc = vfe_core<float>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, &v[0], &v[1], nullptr);
    if (rc) return rc;
    memcpy(value_out, &v[objective], sizeof(float));
  }
  Fp64Problem p(ctx);
  const agp_kernel* k64 = p.params(k, D, mean, noise, N, jitter, M);
  const double* in[3];  // X, Z, y
  rc = p.inputs({{X, N * D}, {Zind, M * D}, {y, N}}, in);
  if (rc) return rc;
  double* out[4];  // noise_diag, mean_diag, z_grad, x_grad
  rc = p.outputs({{noise_diag_out, N}, {mean_diag_out, N}, {z_grad_out, M * D}, {x_grad_out, N * D}}, out);
  if (rc) return rc;
  rc = vfe_grad_impl<double>(ctx, k64, p.mean, p.noise, layout, in[0], N, D, in[1], M, p.jitter, in[2],
                             objective, nullptr, grad_out, out[0], out[1], out[2], out[3]);
  if (rc) return rc;
  return p.narrow();
}

template <typename T>
int vfe_mean_var_impl(agp_vfe_post* p, int layout, const void* Xs, int64_t Ms, void* mean_out, void* var_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (Ms <= 0) return AGP_OK;
  int64_t cap = (int64_t)(2.0e9 / ((double)p->m_pad * sizeof(T)));
  { const int64_t c_env = env_int64("AGP_PREDICT_CHUNK", 0); if (c_env > 0) cap = c_env; }
  cap = cap / TILE * TILE;
  if (cap < TILE) cap = TILE;
  for (int64_t c0 = 0; c0 < Ms; c0 += cap) {
    const int64_t mc = (Ms - c0 < cap) ? (Ms - c0) : cap;
    const int64_t c_pad = round_up(mc, TILE);
    Scratch sc(ctx);
    const void* xs_chunk = (layout == AGP_POINT_MAJOR) ? (const void*)((const char*)Xs + (size_t)c0 * p->D * sizeof(T)) : Xs;
    const int saved_memspace = ctx->memspace;
    if (layout != AGP_POINT_MAJOR && !(c0 == 0 && mc == Ms)) {  // RowVecs test set larger than one chunk
      T* g = nullptr;
      int grc = gather_feature_major_chunk<T>(ctx, sc, Xs, Ms, p->D, c0, mc, &g);
      if (grc) return grc;
      xs_chunk = g;
      ctx->memspace = AGP_MEM_DEVICE;
    }
    T* Xst = nullptr;
    int rc = prep_points<T>(ctx, sc, &p->k, (const T*)p->ard, layout, xs_chunk, mc, c_pad, p->D, &Xst, false);
    ctx->memspace = saved_memspace;
    if (rc) return rc;
    void* tmp = nullptr;
    CK(sc.alloc(&tmp, (size_t)p->m_pad * c_pad * sizeof(T)));
    T* B = (T*)tmp;
    CK(sc.alloc(&tmp, (size_t)c_pad * 2 * sizeof(T)));
    T* mu = (T*)tmp; T* var = mu + c_pad;
    GramParams gp{};
    fill_gram_params<T>(gp, &p->k, 0, 0, p->m, mc, nullptr, nullptr);
    launch_gram<T>((const T*)p->Zt, Xst, p->m_pad, c_pad, p->D, B, p->m_pad, gp, s);
    forward_subst_multi<T>(ctx, (const T*)p->U, p->lda, (const T*)p->Udinv, p->m_pad, B, p->m_pad, c_pad);  // A*
    launch_gemv_t<T>(B, p->m_pad, p->m_pad, mc, (const T*)p->m_e, p->mean_kind, p->mean_c, (const T*)nullptr, mu, s);
    launch_kdiag<T>(Xst, mc, p->D, p->k.family, p->k.variance, p->k.linear_c, var, s);
    launch_colsumsq_acc<T>(B, p->m_pad, p->m_pad, mc, -1.0, var, s);
    forward_subst_multi<T>(ctx, (const T*)p->Lam, p->lda, (const T*)p->Ldinv, p->m_pad, B, p->m_pad, c_pad);
    launch_colsumsq_acc<T>(B, p->m_pad, p->m_pad, mc, 1.0, var, s);
    if (mean_out) { rc = download<T>(ctx, (T*)mean_out + c0, mu, mc, false); if (rc) return rc; }
    if (var_out) { rc = download<T>(ctx, (T*)var_out + c0, var, mc, false); if (rc) return rc; }
    CK(cudaStreamSynchronize(s));
  }
  CK(cudaGetLastError());
  return AGP_OK;
}

// ------------------------------------------------------------------------------------------------
// Multi-GPU fit: one process per GPU, block-column-cyclic tiles on a 1 x Q process grid, NCCL panel
// broadcast over NVLink/NVSwitch, look-ahead so the broadcast of panel k+1 overlaps the bulk of the
// trailing update of panel k.  Column block j (128 columns, all rows + the border rows) lives on
// rank j mod Q as local block j div Q.  Every rank generates only its own Gram columns from the
// replicated points.  (grid_p > 1 is declared in the ABI but not built: on NVSwitch the panel
// broadcast is ~5 % of the factorisation at C4, so the 2-D row/column split buys nothing yet.)
// ------------------------------------------------------------------------------------------------
// ---- full predictive covariance of the approximate posterior, and logpdf / rand of a FiniteGP over it (checked in fp64
// arithmetic up to M = 2304 inducing points and 600 test points, tests/test_gpu_vfe_tensor.py).
//   mean_and_cov(::ApproxPosteriorGP, x*)  /root/reference/src/sparse_approximations.jl:205-210 (cov :187-190):
//   A = U' \ K(z, x*),  m* = m(x*) + A' m_e,  C* = K** - A'A + (Lam' \ A)'(Lam' \ A)
// mode "cov": C* (no noise) is returned.  mode "factor": K** + Sigma* is generated with the noise fused, C* + Sigma* is
// factored in place with (Y - m*)' in the border tile (logpdf, src/finite_gp_projection.jl:306-318) and / or multiplied
// into the caller's normals (rand, :233-240) -- the same tail as post_cond_impl.
template <typename T>
int vfe_cond_impl(agp_vfe_post* p, int layout, const void* Xs, int64_t M, const agp_noise* noise_s, void* mean_out,
                  void* cov_out, const void* Y, int S, void* logpdf_out, const void* Z, int Sz, void* rand_out) {
  agp_ctx* ctx = p->ctx;
  cudaStream_t s = ctx->stream;
  CK(cudaSetDevice(ctx->device));
  if (M <= 0) { ctx->err = "M must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (!Xs) { ctx->err = "Xs is NULL"; return AGP_ERR_INVALID; }
  if (S < 0 || S > TILE) { ctx->err = "number of right-hand sides must be in [0,128]"; return AGP_ERR_UNSUPPORTED; }
  if (S > 0 && (!Y || !logpdf_out)) { ctx->err = "Y/logpdf_out is NULL"; return AGP_ERR_INVALID; }
  if (Sz > 0 && (!Z || !rand_out)) { ctx->err = "Z/out is NULL"; return AGP_ERR_INVALID; }
  const bool factor = (S > 0 || Sz > 0);
  static const agp_noise default_noise{0, 1e-18, nullptr};
  if (factor && !noise_s) noise_s = &default_noise;
  if (factor && noise_s->kind == 1 && !noise_s->v) { ctx->err = "noise vector is NULL"; return AGP_ERR_INVALID; }
  const int64_t c_pad = round_up(M, TILE), ldf = c_pad + TILE;
  const int nblk = (int)(c_pad / TILE);
  Scratch sc(ctx);
  T* Xst = nullptr;
  int rc = prep_points<T>(ctx, sc, &p->k, (const T*)p->ard, layout, Xs, M, c_pad, p->D, &Xst, false);
  if (rc) return rc;
  T *noise_d = nullptr, *Yd = nullptr;
  if (factor && noise_s->kind == 1) { rc = upload<T>(ctx, sc, noise_s->v, M, true, &noise_d); if (rc) return rc; }
  if (S > 0) { rc = upload<T>(ctx, sc, Y, (size_t)M * S, false, &Yd); if (rc) return rc; }
  void* tmp = nullptr;
  CK(sc.alloc(&tmp, (size_t)p->m_pad * c_pad * sizeof(T)));
  T* B = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)c_pad * sizeof(T)));
  T* mu = (T*)tmp;
  CK(cudaMemsetAsync(mu, 0, (size_t)c_pad * sizeof(T), s));
  CK(sc.alloc(&tmp, (size_t)ldf * c_pad * sizeof(T)));
  T* Lf = (T*)tmp;
  GramParams gp{};
  fill_gram_params<T>(gp, &p->k, 0, 0, p->m, M, nullptr, nullptr);
  launch_gram<T>((const T*)p->Zt, Xst, p->m_pad, c_pad, p->D, B, p->m_pad, gp, s);
  forward_subst_multi<T>(ctx, (const T*)p->U, p->lda, (const T*)p->Udinv, p->m_pad, B, p->m_pad, c_pad);  // A
  launch_gemv_t<T>(B, p->m_pad, p->m_pad, M, (const T*)p->m_e, p->mean_kind, p->mean_c, (const T*)nullptr, mu, s);
  GramParams gs{};  // K** (+ Sigma* when factoring), full square: the covariance is returned whole
  fill_gram_params<T>(gs, &p->k, 1, 0, M, M, factor ? noise_s : nullptr, noise_d);
  launch_gram<T>(Xst, Xst, c_pad, c_pad, p->D, Lf, ldf, gs, s);
  {
    GemmArgs g{};  // -= A'A
    g.A = B; g.lda = p->m_pad; g.a_kmajor = 1;
    g.B = B; g.ldb = p->m_pad; g.b_kmajor = 1;
    g.C = Lf; g.ldc = ldf; g.M = c_pad; g.N = c_pad; g.K = p->m_pad; g.alpha_neg = 1; g.beta_one = 1;
    launch_gemm<T>(g, s);
  }
  forward_subst_multi<T>(ctx, (const T*)p->Lam, p->lda, (const T*)p->Ldinv, p->m_pad, B, p->m_pad, c_pad);  // Lam' \ A
  {
    GemmArgs g{};  // += (Lam' \ A)'(Lam' \ A)
    g.A = B; g.lda = p->m_pad; g.a_kmajor = 1;
    g.B = B; g.ldb = p->m_pad; g.b_kmajor = 1;
    g.C = Lf; g.ldc = ldf; g.M = c_pad; g.N = c_pad; g.K = p->m_pad; g.beta_one = 1;
    launch_gemm<T>(g, s);
  }
  if (mean_out) { rc = download<T>(ctx, mean_out, mu, (size_t)M, false); if (rc) return rc; }
  if (!factor) {
    if (cov_out) {
      cudaMemcpyKind kind = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
      CK(cudaMemcpy2DAsync(cov_out, (size_t)M * sizeof(T), Lf, (size_t)ldf * sizeof(T), (size_t)M * sizeof(T), (size_t)M, kind, s));
    }
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    return AGP_OK;
  }
  CK(sc.alloc(&tmp, (size_t)nblk * TILE * TILE * sizeof(T)));
  T* Dinv = (T*)tmp;
  CK(sc.alloc(&tmp, (size_t)(nblk + TILE + 2) * sizeof(double)));
  double* dscal = (double*)tmp;
  CK(sc.alloc(&tmp, sizeof(int)));
  int* dinfo = (int*)tmp;
  CK(cudaMemsetAsync(dinfo, 0, sizeof(int), s));
  CK(sc.alloc(&tmp, (size_t)TILE * sizeof(T)));
  T* lp_d = (T*)tmp;
  launch_border_init<T>(Lf, ldf, M, c_pad, Yd, M, S, 2, 0.0, (const T*)mu, s);  // border = (Y - m*)'
  prof_begin(ctx);
  cholesky_inplace<T>(ctx, Lf, ldf, c_pad, ldf, Dinv, dscal, dinfo);
  if (S > 0) {
    CK(sc.alloc(&tmp, (size_t)S * c_pad * sizeof(T)));
    launch_extract_v<T>(Lf, ldf, c_pad, S, (T*)tmp, dscal + nblk, s);
    launch_finalize_logpdf<T>(dscal, nblk, dscal + nblk, S, M, lp_d, dscal + nblk + TILE, s);
  }
  int h_info = 0;
  CK(cudaMemcpyAsync(&h_info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (h_info != 0) {
    ctx->info = h_info;
    char b[128];
    snprintf(b, sizeof(b), "approximate posterior covariance is not positive definite; Cholesky failed at pivot %d", h_info);
    ctx->err = b;
    return AGP_ERR_NOT_POSDEF;
  }
  if (S > 0) CK(cudaMemcpyAsync(logpdf_out, lp_d, (size_t)S * sizeof(T), cudaMemcpyDeviceToHost, s));
  if (Sz > 0) {
    const int64_t s_pad = round_up(Sz, 4);
    CK(sc.alloc(&tmp, (size_t)c_pad * s_pad * sizeof(T) * 2));
    T* Zd = (T*)tmp; T* Od = Zd + c_pad * s_pad;
    CK(cudaMemsetAsync(Zd, 0, (size_t)c_pad * s_pad * sizeof(T), s));
    cudaMemcpyKind kin = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    cudaMemcpyKind kout = ctx->memspace == AGP_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    CK(cudaMemcpy2DAsync(Zd, (size_t)c_pad * sizeof(T), Z, (size_t)M * sizeof(T), (size_t)M * sizeof(T), (size_t)Sz, kin, s));
    GemmArgs g{};
    g.A = Lf; g.lda = ldf; g.a_kmajor = 0;
    g.B = Zd; g.ldb = c_pad; g.b_kmajor = 1;
    g.C = Od; g.ldc = c_pad; g.M = c_pad; g.N = s_pad; g.K = c_pad; g.trmm_lower = 1;
    launch_gemm<T>(g, s);
    launch_add_mean_cols<T>(Od, c_pad, M, Sz, 2, 0.0, (const T*)mu, s);
    CK(cudaMemcpy2DAsync(rand_out, (size_t)M * sizeof(T), Od, (size_t)c_pad * sizeof(T), (size_t)M * sizeof(T), (size_t)Sz, kout, s));
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return AGP_OK;
}

template <typename T>
int fit_dist_impl(agp_ctx* ctx, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise, int layout,
                  const void* X, int64_t N, int D, const void* Y, int S, void* logpdf_out, void* alpha_out,
                  agp_post** post_out) {
  int rc = check_kernel(ctx, k, D);
  if (rc) return rc;
  if (N <= 0) { ctx->err = "N must be positive"; return AGP_ERR_DIM_MISMATCH; }
  if (S < 1 || S > TILE || !Y) { ctx->err = "distributed fit needs 1..128 right-hand sides"; return AGP_ERR_UNSUPPORTED; }
  const bool keep = post_out != nullptr;
  static const agp_mean zero_mean{0, 0.0, nullptr};
  static const agp_noise default_noise{0, 1e-18, nullptr};
  if (!mean) mean = &zero_mean;
  if (!noise) noise = &default_noise;
  cudaStream_t s = ctx->stream, s2 = ctx->stream2;
  CK(cudaSetDevice(ctx->device));
  Scratch sc(ctx);
  const int R = ctx->nranks, me = ctx->rank;
  // distribution block = one OUTER panel of G inner 128-blocks (W columns): the owner factors it locally,
  // one NCCL broadcast per outer panel, rank-W trailing updates
  const int G = resolve_G(ctx, round_up(N, TILE));
  const int64_t W = (int64_t)G * TILE;
  const int64_t n_pad = round_up(N, W), lda = n_pad + TILE;
  const int nto = (int)(n_pad / W), nt = (int)(n_pad / TILE);
  const int nloc = (nto - me + R - 1) / R;  // local outer blocks: global jo = ljo * R + me
  const int fp64_mode = resolve_fp64_mode(ctx, n_pad);
  prof_begin(ctx);
  CK(cudaEventRecord(ctx->ev[0], s));
  // big buffers FIRST (the local block columns, then the packed panels): the pool returns the blocks the previous fit freed
  // before the small staging buffers can split them (see fit_impl)
  void *Lv = nullptr, *Dv = nullptr, *Pv = nullptr;
  CK(cudaMallocAsync(&Lv, (size_t)lda * (nloc > 0 ? nloc : 1) * W * sizeof(T), s));
  struct BufGuard { void* p; cudaStream_t s; ~BufGuard() { if (p) cudaFreeAsync(p, s); } } lguard{Lv, s};
  CK(sc.alloc(&Pv, (size_t)3 * lda * W * sizeof(T)));
  T *ard_d = nullptr, *mean_d = nullptr, *noise_d = nullptr, *Yd = nullptr, *Xt = nullptr;
  if (k->transform == AGP_T_ARD) { rc = upload<T>(ctx, sc, k->ard, D, true, &ard_d); if (rc) return rc; }
  if (mean->kind == 2) { rc = upload<T>(ctx, sc, mean->v, N, true, &mean_d); if (rc) return rc; }
  if (noise->kind == 1) { rc = upload<T>(ctx, sc, noise->v, N, true, &noise_d); if (rc) return rc; }
  rc = upload<T>(ctx, sc, Y, (size_t)N * S, false, &Yd); if (rc) return rc;
  rc = prep_points<T>(ctx, sc, k, ard_d, layout, X, N, n_pad, D, &Xt, keep); if (rc) return rc;
  CK(cudaEventRecord(ctx->ev[1], s));
  void* tmp = nullptr;
  // the factor and its inverse diagonal blocks outlive the call when a posterior handle is requested
  agp_post* post = nullptr;
  lguard.p = nullptr;  // ownership passes to the handle / scratch list below
  CK(cudaMallocAsync(&Dv, (size_t)(nloc > 0 ? nloc : 1) * G * TILE * TILE * sizeof(T), s));
  if (keep) {
    post = new agp_post();
    post->ctx = ctx; post->dtype = sizeof(T) == 8 ? AGP_F64 : AGP_F32;
    post->n = N; post->n_pad = n_pad; post->lda = lda; post->D = D;
    post->Lloc = Lv; post->Dinv_loc = Dv; post->Xt = Xt;
    post->dist_R = R; post->dist_me = me; post->dist_G = G; post->dist_nloc = nloc; post->dist_W = W;
    post->k = *k; post->k.ard = nullptr;
    post->mean_kind = mean->kind == 2 ? 0 : mean->kind; post->mean_c = mean->c;
    post->segs.push_back({0, N});
    if (ard_d) { sc.release(ard_d); post->ard = ard_d; }
  } else {
    sc.ptrs.push_back(Lv); sc.ptrs.push_back(Dv);
  }
  struct PostGuard { agp_post* p; ~PostGuard() { if (p) agp_post_free(p); } } guard{post};  // freed on every error return
  T* L = (T*)Lv;
  T* Dinv = (T*)Dv;  // inverse diagonal blocks of the LOCAL 128-blocks
  T* P[3] = {(T*)Pv, (T*)Pv + lda * W, (T*)Pv + 2 * lda * W};  // packed panels (rows_below x W, ld = rows_below): two in
                                                                   // flight in the default schedule, three in the pipelined one
  CK(sc.alloc(&tmp, (size_t)(nt + TILE + 4) * sizeof(double)));
  double* dscal = (double*)tmp;  // [0..nt) logdet parts, [nt..nt+TILE) sqmahal, [nt+TILE] logdet
  CK(cudaMemsetAsync(dscal, 0, (size_t)(nt + TILE + 4) * sizeof(double), s));
  CK(sc.alloc(&tmp, sizeof(int)));
  int* dinfo = (int*)tmp;
  CK(cudaMemsetAsync(dinfo, 0, sizeof(int), s));
  CK(sc.alloc(&tmp, (size_t)(S + 1) * n_pad * sizeof(T)));
  T* rwork = (T*)tmp; T* alpha = rwork + (size_t)S * n_pad;
  CK(cudaMemsetAsync(rwork, 0, (size_t)(S + 1) * n_pad * sizeof(T), s));
  CK(sc.alloc(&tmp, (size_t)TILE * sizeof(T)));
  T* lp_d = (T*)tmp;
  const OzakiWs* oz = nullptr;
  if constexpr (std::is_same<T, double>::value) {
    if (fp64_mode == 1 && nto > 2 && W % 64 == 0) {
      if (ensure_oz<T>(ctx, lda, (int)W, true, s)) oz = &ctx->oz;
    }
  }
  // schedule: 2 = pipelined (default for R > 1; see the loop below), 1 = round-1 owner-first experiment, 0 = plain look-ahead
  int dist_sched = (R > 1) ? 2 : 0;
  { const char* e1 = getenv("AGP_DIST_SCHED"); if (e1) dist_sched = atoi(e1); }
  const OzakiWs* oz_b = nullptr;  // second slice buffer (pipelined schedule only)
  if constexpr (std::is_same<T, double>::value) {
    if (dist_sched == 2 && oz) {
      oz_b = ensure_oz2<T>(ctx, lda, (int)W, true, s) ? &ctx->oz2 : nullptr;
      if (!oz_b) dist_sched = 0;
    }
  }
  if (dist_sched == 2 && !ctx->stream_comm) {
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    CK(cudaStreamCreateWithPriority(&ctx->stream_comm, cudaStreamNonBlocking, prio_hi));
  }

  // ---- Gram: only the local outer blocks, lower part, + border rows
  for (int lj = 0; lj < nloc; ++lj) {
    const int64_t jo = (int64_t)lj * R + me;
    GramParams gp{};
    fill_gram_params<T>(gp, k, 1, 1, N, N, noise, noise_d);
    gp.diag_off = jo * W;
    T* col = L + (int64_t)lj * W * lda;
    launch_gram<T>(Xt, Xt + jo * W * D, n_pad, W, D, col, lda, gp, s);
    launch_border_init_cols<T>(col, lda, n_pad, jo * W, W, N, Yd, N, S, mean->kind, mean->c, mean_d, s);
  }
  CK(cudaEventRecord(ctx->ev[2], s));

  // ---- distributed right-looking Cholesky with look-ahead
  auto local_first_after = [&](int kk) {  // first local outer block whose global index > kk
    int lj = (kk + 1 - me + R - 1) / R;
    if (lj < 0) lj = 0;
    while ((int64_t)lj * R + me <= kk) ++lj;
    return lj;
  };
  const OzakiWs* oz_cur = oz;  // slice buffer the `trailing` launches read (the pipelined schedule alternates two)
  auto trailing = [&](int kk, T* Pk, int lj_lo, int lj_hi, bool use_oz, cudaStream_t st) {  // local outer blocks [lj_lo, lj_hi)
    if (lj_lo >= lj_hi) return;
    const int64_t rows_below = lda - (int64_t)(kk + 1) * W;
    const int64_t j0 = (int64_t)lj_lo * R + me;
    T* C = L + (int64_t)(kk + 1) * W + (int64_t)lj_lo * W * lda;
    const int64_t Ncols = (int64_t)(lj_hi - lj_lo) * W, b_off = (j0 - (kk + 1)) * W;
    if (ctx->profile) cudaEventRecord(prof_event(ctx), st);
    bool done = false;
    if constexpr (std::is_same<T, double>::value) {
      if (use_oz) done = ozaki_syrk(*oz_cur, C, lda, rows_below, Ncols, 1, (int64_t)R * W, W, b_off, 0, st) == 0;
    }
    if (!done) {
      GemmArgs u{};
      u.A = Pk; u.lda = rows_below; u.B = Pk; u.ldb = rows_below; u.C = C; u.ldc = lda;
      u.M = rows_below; u.N = Ncols; u.K = W; u.alpha_neg = 1; u.beta_one = 1; u.lower_only = 1;
      u.b_tile_stride = (int64_t)R * W; u.b_tile_width = W; u.b_off = b_off;
      launch_gemm<T>(u, st);
    }
    if (ctx->profile) cudaEventRecord(prof_event(ctx), st);
  };
  bool rest_pending = false;
  size_t ev_idx = 0, last_rest = 0;
  // EXPERIMENTAL schedule (AGP_DIST_SCHED=1, not yet validated on a multi-GPU box; default off).  The persistent
  // update kernel holds every SM until it ends, so in the default order the next panel's owner factors it only
  // AFTER its own rest update and every peer's broadcast kernel starts only after theirs: the step costs
  // rest + factor + broadcast.  Here (1) the owner of panel kk+1 defers its rest update of step kk until panel kk+1
  // is factored and packed (the broadcast is enqueued right behind), and (2) rest updates run on nsm - reserve
  // CTAs so that the NCCL kernels of the next broadcast find SMs while the update is still running.
  bool sched2 = false;
  int reserve_sms = 16;
  if (R > 1) {
    sched2 = dist_sched == 1;
    const char* e2 = getenv("AGP_DIST_RESERVE_SMS");
    if (e2) reserve_sms = atoi(e2);
    if (reserve_sms < 0 || reserve_sms > 64) reserve_sms = 16;
  }
  // pipelined schedule: 1 = the owner of the next panel runs its rest update AFTER that panel's factorisation; 0 = at once
  // (bounded CTAs + stream priorities let the factorisation through)
  const bool dist_defer = env_int64("AGP_DIST_DEFER", 1) != 0;
  int nsm_dev = 0;
  cudaDeviceGetAttribute(&nsm_dev, cudaDevAttrMultiProcessorCount, ctx->device);
  struct DeferredRest { bool on; int kk; T* Pk; int lo, hi; bool use_oz; cudaEvent_t e_rest; };
  DeferredRest def{false, 0, nullptr, 0, 0, false, nullptr};
  auto rest_update = [&](int kk, T* Pk, int lo, int hi, bool use_oz, cudaEvent_t e_rest) {
    if (oz && sched2) oz->max_ctas = nsm_dev - reserve_sms;
    trailing(kk, Pk, lo, hi, use_oz, s2);
    if (oz) oz->max_ctas = 0;
    cudaEventRecord(e_rest, s2);
  };
  if (dist_sched == 2) {
    // ---- PIPELINED schedule.  The critical path of a 1 x R factorisation is the owner chain
    //   [panel k-1 received] -> update of block column k -> factor panel k -> broadcast panel k,
    // so (1) the owner factors its panel BEFORE its own rest update of the previous step (deferred to stream2 behind the
    // factorisation); (2) the panel is broadcast in G column pieces on a communication stream, each as soon as its inner
    // block is final, so only the last piece is exposed; (3) rest updates leave `reserve_sms` SMs to the NCCL kernels;
    // (4) panels rotate through three buffers and slices through two, so receiving / slicing panel k+1 never waits for
    // the rest update of step k.  Every rank issues the same collectives in the same order on stream_comm; the
    // collectives that follow the factorisation are issued after the streams are joined.
    cudaStream_t scm = ctx->stream_comm;
    std::vector<cudaEvent_t> e_rest((size_t)nto, nullptr), e_first((size_t)nto, nullptr);
    auto ev = [&]() { return dep_event(ctx, ev_idx++); };
    cudaEvent_t e_start = ev();
    cudaEventRecord(e_start, s);
    cudaStreamWaitEvent(scm, e_start, 0);  // the Gram (and the previous call) precede the first broadcast
    cudaStreamWaitEvent(s2, e_start, 0);
    struct Deferred { bool on; int kk; T* Pk; int lo, hi; bool use_oz; const OzakiWs* ws; cudaEvent_t e_prep; } dfr{false, 0, nullptr, 0, 0, false, nullptr, nullptr};
    auto issue_rest = [&](int kk, T* Pk, int lo, int hi, bool use_oz, const OzakiWs* ws) {
      e_rest[(size_t)kk] = ev();
      if (ws) { ws->max_ctas = nsm_dev - reserve_sms; ws->chunk_tiles = ctx->oz_chunk; }
      oz_cur = ws;
      // The rank that owns block column kk+2 will update it on the MAIN stream at step kk+1 (next-panel update) and then
      // factor it: this rest update must have finished with that column before.  It is the first local block of the
      // range (the rank does not own kk+1), so it goes first, alone, with its own event -- the chain of step kk+1 waits
      // for this piece only, not for the whole rest update.
      if (kk + 2 < nto && (kk + 2) % R == me && hi > lo) {
        e_first[(size_t)kk] = ev();
        trailing(kk, Pk, lo, lo + 1, use_oz, s2);
        cudaEventRecord(e_first[(size_t)kk], s2);
        trailing(kk, Pk, lo + 1, hi, use_oz, s2);
      } else {
        trailing(kk, Pk, lo, hi, use_oz, s2);
      }
      if (ws) { ws->max_ctas = 0; ws->chunk_tiles = 0; }
      cudaEventRecord(e_rest[(size_t)kk], s2);
    };
    for (int kk = 0; kk < nto; ++kk) {
      const int owner = kk % R;
      const int64_t rows_below = lda - (int64_t)(kk + 1) * W;
      T* Pk = P[kk % 3];
      const OzakiWs* ws_k = (kk & 1) ? oz_b : oz;
      if (kk >= 3 && e_rest[(size_t)kk - 3]) cudaStreamWaitEvent(scm, e_rest[(size_t)kk - 3], 0);  // P[kk % 3] is free again
      if (owner == me) {
        const int lk = kk / R;
        T* Lp = L + (int64_t)kk * W + (int64_t)lk * W * lda;
        if (kk >= 3 && e_rest[(size_t)kk - 3]) cudaStreamWaitEvent(s, e_rest[(size_t)kk - 3], 0);  // the pack below writes P[kk % 3]
        for (int g = 0; g < G; ++g) {
          // inner block g of the panel: rows from the panel's diagonal block down to the border
          factor_panel_step<T>(ctx, Lp, lda, G, g, lda - (int64_t)kk * W, Dinv + (int64_t)lk * G * TILE * TILE, dscal, kk * G, dinfo, s);
          launch_copy2d<T>(Lp + W + (int64_t)g * TILE * lda, lda, Pk + (int64_t)g * TILE * rows_below, rows_below, rows_below, TILE, s);
          cudaEvent_t e_col = ev();
          cudaEventRecord(e_col, s);
          cudaStreamWaitEvent(scm, e_col, 0);
          if (rows_below > 0)
            CKN(ncclBroadcast(Pk + (int64_t)g * TILE * rows_below, Pk + (int64_t)g * TILE * rows_below, (size_t)rows_below * TILE,
                              NcclType<T>::v, owner, ctx->nccl, scm));
        }
        if (dfr.on) {  // this rank's rest update of step kk-1, behind the factorisation it must not delay
          cudaEvent_t e_fact = ev();
          cudaEventRecord(e_fact, s);
          cudaStreamWaitEvent(s2, e_fact, 0);
          issue_rest(dfr.kk, dfr.Pk, dfr.lo, dfr.hi, dfr.use_oz, dfr.ws);
          dfr.on = false;
        }
      } else if (rows_below > 0) {
        for (int g = 0; g < G; ++g)
          CKN(ncclBroadcast(Pk + (int64_t)g * TILE * rows_below, Pk + (int64_t)g * TILE * rows_below, (size_t)rows_below * TILE,
                            NcclType<T>::v, owner, ctx->nccl, scm));
      }
      if (kk == nto - 1) break;
      cudaEvent_t e_recv = ev();
      cudaEventRecord(e_recv, scm);
      cudaStreamWaitEvent(s, e_recv, 0);
      if (kk >= 2 && e_rest[(size_t)kk - 2]) cudaStreamWaitEvent(s, e_rest[(size_t)kk - 2], 0);  // slice buffer kk & 1 is free again
      bool use_oz = false;
      if constexpr (std::is_same<T, double>::value) {
        if (ws_k && (int64_t)(nto - 1 - kk) * W >= 2 * TILE) {
          ozaki_prepare(*ws_k, (const double*)Pk, rows_below, rows_below, s);
          use_oz = true;
        }
      }
      cudaEvent_t e_prep = ev();
      cudaEventRecord(e_prep, s);
      const int lj_first = local_first_after(kk);
      int lj_bulk = lj_first;
      const bool next_is_mine = (kk + 1) % R == me;
      if (next_is_mine) {  // the next panel's block column first, on the main stream; its factorisation follows
        if (kk >= 1 && e_first[(size_t)kk - 1]) cudaStreamWaitEvent(s, e_first[(size_t)kk - 1], 0);  // see issue_rest
        else if (kk >= 1 && e_rest[(size_t)kk - 1]) cudaStreamWaitEvent(s, e_rest[(size_t)kk - 1], 0);
        oz_cur = ws_k;
        trailing(kk, Pk, lj_first, lj_first + 1, use_oz, s);
        lj_bulk = lj_first + 1;
      }
      if (next_is_mine && dist_defer) {
        dfr = Deferred{true, kk, Pk, lj_bulk, nloc, use_oz, use_oz ? ws_k : nullptr, e_prep};
      } else {
        cudaStreamWaitEvent(s2, e_prep, 0);
        issue_rest(kk, Pk, lj_bulk, nloc, use_oz, use_oz ? ws_k : nullptr);
      }
    }
    if (dfr.on) {  // cannot happen (the last step has no trailing work), kept for safety
      cudaStreamWaitEvent(s2, dfr.e_prep, 0);
      issue_rest(dfr.kk, dfr.Pk, dfr.lo, dfr.hi, dfr.use_oz, dfr.ws);
    }
    cudaEvent_t e_s2 = ev(), e_cm = ev();
    cudaEventRecord(e_s2, s2);
    cudaEventRecord(e_cm, scm);
    cudaStreamWaitEvent(s, e_s2, 0);
    cudaStreamWaitEvent(s, e_cm, 0);
    oz_cur = oz;
  } else
  for (int kk = 0; kk < nto; ++kk) {
    const int owner = kk % R;
    const int64_t rows_below = lda - (int64_t)(kk + 1) * W;
    T* Pk = P[kk & 1];
    if (owner == me) {
      const int lk = kk / R;
      T* Lp = L + (int64_t)kk * W + (int64_t)lk * W * lda;
      factor_panel<T>(ctx, Lp, lda, G, lda - (int64_t)kk * W, Dinv + (int64_t)lk * G * TILE * TILE, dscal, kk * G, dinfo, s);
      launch_copy2d<T>(Lp + W, lda, Pk, rows_below, rows_below, W, s);
    }
    if (def.on) {  // this rank owns panel kk and still owes step kk-1's rest update: it goes behind the factorisation
      cudaEvent_t e_fact = dep_event(ctx, ev_idx++);
      cudaEventRecord(e_fact, s);
      cudaStreamWaitEvent(s2, e_fact, 0);
      rest_update(def.kk, def.Pk, def.lo, def.hi, def.use_oz, def.e_rest);
      def.on = false;
    }
    if (R > 1) CKN(ncclBroadcast(Pk, Pk, (size_t)rows_below * W, NcclType<T>::v, owner, ctx->nccl, s));
    if (kk == nto - 1) break;
    if (rest_pending) cudaStreamWaitEvent(s, dep_event(ctx, last_rest), 0);  // frees P[(kk+1)&1] and the slice buffer
    bool use_oz = false;
    if constexpr (std::is_same<T, double>::value) {
      if (oz && (int64_t)(nto - 1 - kk) * W >= 2 * TILE) {
        ozaki_prepare(*oz, (const double*)Pk, rows_below, rows_below, s);
        use_oz = true;
      }
    }
    cudaEvent_t e_panel = dep_event(ctx, ev_idx++), e_rest = dep_event(ctx, ev_idx++);
    cudaEventRecord(e_panel, s);
    const int lj_first = local_first_after(kk);
    int lj_bulk = lj_first;
    if ((kk + 1) % R == me) {  // next panel first (only its owner has it), on the main stream
      trailing(kk, Pk, lj_first, lj_first + 1, use_oz, s);
      lj_bulk = lj_first + 1;
    }
    rest_pending = true;
    last_rest = ev_idx - 1;  // index of e_rest
    if (sched2 && (kk + 1) % R == me) {
      def = DeferredRest{true, kk, Pk, lj_bulk, nloc, use_oz, e_rest};  // launched at the top of the next iteration
    } else {
      cudaStreamWaitEvent(s2, e_panel, 0);
      rest_update(kk, Pk, lj_bulk, nloc, use_oz, e_rest);
    }
  }
  if (rest_pending) cudaStreamWaitEvent(s, dep_event(ctx, last_rest), 0);
  join_inverses(ctx);
  CK(cudaEventRecord(ctx->ev[3], s));

  // ---- v = border rows (distributed by column), sqmahal and logdet via all-reduce
  for (int lj = 0; lj < nloc; ++lj) {
    const int64_t jo = (int64_t)lj * R + me;
    for (int sI = 0; sI < S; ++sI)
      launch_copy2d<T>(L + n_pad + sI + (int64_t)lj * W * lda, lda, rwork + (size_t)sI * n_pad + jo * W, 1, 1, W, s);
  }
  for (int sI = 0; sI < S; ++sI) launch_sumsq<T>(rwork + (size_t)sI * n_pad, n_pad, dscal + nt + sI, s);
  if (R > 1) CKN(ncclAllReduce(dscal, dscal, (size_t)(nt + TILE), ncclDouble, ncclSum, ctx->nccl, s));
  // ---- distributed backward substitution for column 0: alpha = L^-T v.  The owner of an outer block holds its G diagonal
  // blocks and every tile between them, so it resolves the whole block in ONE single-CTA kernel; ONE broadcast per outer
  // block ships G*128 values (128 collectives at C4).  The critical chain per block is
  //   [alpha of block io+1 arrives] -> update of block io only (G CTAs) -> block solve -> broadcast;
  // the bulk update of the other local columns with block io+1's alpha runs behind the broadcast on the owner and before it
  // on the other ranks (who would otherwise idle in the collective).
  {
    int pending = -1;  // outer block whose alpha has been received but not yet applied to (all of) the local columns
    for (int io = nto - 1; io >= 0; --io) {
      const int owner = io % R, i_lo = io * G;
      const int64_t p_lo = (int64_t)(pending >= 0 ? pending : 0) * G;
      T* a_pend = alpha + p_lo * TILE;
      if (owner == me) {
        if (pending >= 0)  // own block first
          launch_bwd_update_local_multi<T>(L, lda, (int)p_lo, G, a_pend, rwork, nloc * G, me, R, G, i_lo, (int64_t)i_lo + G, s);
        launch_bwd_block_solve<T>(L + (int64_t)io * W + (int64_t)(io / R) * W * lda, lda, Dinv + (int64_t)(io / R) * G * TILE * TILE,
                                  rwork + (int64_t)i_lo * TILE, alpha + (int64_t)i_lo * TILE, G, s);
      } else if (pending >= 0) {
        launch_bwd_update_local_multi<T>(L, lda, (int)p_lo, G, a_pend, rwork, nloc * G, me, R, G, 0, p_lo, s);
      }
      // alpha is zero on every rank but the owner (the buffer starts zeroed and only owners write their blocks), so an
      // all-reduce(sum) IS the broadcast -- and its small-message latency (tree / NVLS) does not grow with the ring length
      // like ncclBroadcast's (measured 0.17 ms per block at 8 ranks with the broadcast)
      if (R > 1) CKN(ncclAllReduce(alpha + (int64_t)i_lo * TILE, alpha + (int64_t)i_lo * TILE, (size_t)G * TILE, NcclType<T>::v, ncclSum, ctx->nccl, s));
      if (owner == me && pending >= 0)
        launch_bwd_update_local_multi<T>(L, lda, (int)p_lo, G, a_pend, rwork, nloc * G, me, R, G, 0, i_lo, s);
      pending = io;
    }
  }
  launch_finalize_logpdf<T>(dscal, nt, dscal + nt, S, N, lp_d, dscal + nt + TILE, s);
  CK(cudaEventRecord(ctx->ev[4], s));
  int h_info = 0;
  if (R > 1) CKN(ncclAllReduce(dinfo, dinfo, 1, ncclInt, ncclMax, ctx->nccl, s));
  CK(cudaMemcpyAsync(&h_info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, s));
  if (logpdf_out) CK(cudaMemcpyAsync(logpdf_out, lp_d, (size_t)S * sizeof(T), cudaMemcpyDeviceToHost, s));
  if (alpha_out) { rc = download<T>(ctx, alpha_out, alpha, (size_t)N, false); if (rc) return rc; }
  CK(cudaEventRecord(ctx->ev[5], s));
  CK(cudaStreamSynchronize(s));
  CK(cudaStreamSynchronize(s2));
  CK(cudaGetLastError());
  float ms = 0;
  auto el = [&](int a, int b) { cudaEventElapsedTime(&ms, ctx->ev[a], ctx->ev[b]); return (double)ms; };
  ctx->timings[0] = el(0, 5); ctx->timings[1] = el(0, 1); ctx->timings[2] = el(1, 2); ctx->timings[3] = el(2, 3);
  ctx->timings[4] = el(3, 4); ctx->timings[5] = el(4, 5); ctx->timings[6] = 0.0;
  ctx->timings[7] = ctx->profile ? prof_total_ms(ctx) : 0.0;
  if (h_info != 0) {
    ctx->info = h_info;
    ctx->err = "matrix is not positive definite (distributed Cholesky)";
    return AGP_ERR_NOT_POSDEF;
  }
  if (keep) {  // alpha, delta = y - m (first column) and log det move into the handle
    CK(cudaMallocAsync(&post->alpha, (size_t)n_pad * sizeof(T), s));
    CK(cudaMallocAsync(&post->delta, (size_t)n_pad * sizeof(T), s));
    CK(cudaMemcpyAsync(post->alpha, alpha, (size_t)n_pad * sizeof(T), cudaMemcpyDeviceToDevice, s));
    CK(cudaMemsetAsync(post->delta, 0, (size_t)n_pad * sizeof(T), s));
    launch_sub_mean<T>(Yd, N, mean->kind, mean->c, mean_d, (T*)post->delta, s);
    double h_logdet = 0.0;
    CK(cudaMemcpyAsync(&h_logdet, dscal + nt + TILE, sizeof(double), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    post->logdet = h_logdet;
    guard.p = nullptr;
    *post_out = post;
  }
  return AGP_OK;
}

int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// extern "C" ABI
// ------------------------------------------------------------------------------------------------
#define DISPATCH(dtype, call_f32, call_f64)                                   \
  ((dtype) == AGP_F32 ? (call_f32) : ((dtype) == AGP_F64 ? (call_f64) : (int)AGP_ERR_UNSUPPORTED))

extern "C" {

const char* agp_version(void) { return "agp-blackwell 0.1 (sm_90a)"; }

int32_t agp_init(agp_ctx** out, int32_t device, const agp_config* cfg) {
  if (!out) return AGP_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return AGP_ERR_CUDA;  // no CPU fallback, by design
  if (device < 0 || device >= ndev) return AGP_ERR_INVALID;
  agp_ctx* ctx = new agp_ctx();
  ctx->device = device;
  if (cfg) ctx->cfg = *cfg;
  ctx->cfg.tile_nb = env_int("AGP_NB", (cfg && cfg->tile_nb > 0) ? cfg->tile_nb : 0);  // 0 = auto
  if (ctx->cfg.tile_nb % TILE) ctx->cfg.tile_nb = 0;
  ctx->cfg.fp64_mode = env_int("AGP_FP64_MODE", cfg ? ctx->cfg.fp64_mode : -1);            // -1 = auto
  ctx->cfg.fp32_mode = env_int("AGP_FP32_MODE", cfg ? ctx->cfg.fp32_mode : -1);            // -1 = auto
  ctx->cfg.lookahead = env_int("AGP_LOOKAHEAD", cfg ? ctx->cfg.lookahead : 2);  // 2: depth-2 look-ahead on the DMMA path
  ctx->cfg.use_graph = env_int("AGP_GRAPH", ctx->cfg.use_graph);
  ctx->profile = env_int("AGP_PROFILE", cfg ? cfg->profile_kernels : 0);
  ctx->oz_S = env_int("AGP_OZAKI_S", (cfg && cfg->ozaki_slices) ? cfg->ozaki_slices : 6);
  if (ctx->oz_S < 5 || ctx->oz_S > 8) ctx->oz_S = 6;
  ctx->oz_S32 = env_int("AGP_OZAKI_S32", 4);
  if (ctx->oz_S32 < 3 || ctx->oz_S32 > 5) ctx->oz_S32 = 4;
  if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return AGP_ERR_CUDA; }
  // priorities: the panel chain (main stream), the strip inverses and the panel broadcasts go first; the bulk trailing
  // updates (stream2, bounded CTAs) fill whatever SMs are left -- block scheduling honours stream priority
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess) { delete ctx; return AGP_ERR_CUDA; }
  if (cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, prio_lo) != cudaSuccess) { delete ctx; return AGP_ERR_CUDA; }
  if (cudaStreamCreateWithPriority(&ctx->stream3, cudaStreamNonBlocking, prio_hi) != cudaSuccess) { delete ctx; return AGP_ERR_CUDA; }
  ctx->oz_chunk = env_int("AGP_OZAKI_CHUNK", 16);
  if (ctx->oz_chunk < 0 || ctx->oz_chunk > 4096) ctx->oz_chunk = 16;
  cudaEventCreateWithFlags(&ctx->ev_s3, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&ctx->ev_fac, cudaEventDisableTiming);
  for (int i = 0; i < 8; ++i) cudaEventCreate(&ctx->ev[i]);
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = UINT64_MAX;  // keep freed blocks: repeated fits of the same size never hit the OS
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  *out = ctx;
  return AGP_OK;
}

int32_t agp_destroy(agp_ctx* ctx) {
  if (!ctx) return AGP_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (int i = 0; i < 8; ++i) cudaEventDestroy(ctx->ev[i]);
  for (auto e : ctx->prof_ev) cudaEventDestroy(e);
  for (auto e : ctx->dep_ev) cudaEventDestroy(e);
  if (ctx->oz.SL) ozaki_ws_destroy(&ctx->oz, ctx->stream);
  if (ctx->oz2.SL) ozaki_ws_destroy(&ctx->oz2, ctx->stream);
  if (ctx->ozp.SL) ozaki_ws_destroy(&ctx->ozp, ctx->stream);
  if (ctx->stream_comm) { cudaStreamSynchronize(ctx->stream_comm); cudaStreamDestroy(ctx->stream_comm); }
  if (ctx->nccl) ncclCommDestroy(ctx->nccl);
  cudaEventDestroy(ctx->ev_s3);
  cudaEventDestroy(ctx->ev_fac);
  cudaStreamDestroy(ctx->stream3);
  cudaStreamDestroy(ctx->stream2);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
  return AGP_OK;
}

const char* agp_last_error(const agp_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }
int64_t agp_last_info(const agp_ctx* ctx) { return ctx ? ctx->info : 0; }
int32_t agp_set_memspace(agp_ctx* ctx, int32_t m) {
  if (!ctx || (m != AGP_MEM_HOST && m != AGP_MEM_DEVICE)) return AGP_ERR_INVALID;
  ctx->memspace = m;
  return AGP_OK;
}
int32_t agp_set_config(agp_ctx* ctx, const agp_config* cfg) {
  if (!ctx || !cfg) return AGP_ERR_INVALID;
  if (cfg->tile_nb < 0 || cfg->tile_nb % TILE) return AGP_ERR_INVALID;
  ctx->cfg.tile_nb = cfg->tile_nb;
  ctx->cfg.fp64_mode = cfg->fp64_mode;
  ctx->cfg.fp32_mode = cfg->fp32_mode;
  ctx->cfg.lookahead = cfg->lookahead;
  ctx->profile = cfg->profile_kernels;
  if (cfg->ozaki_slices >= 5 && cfg->ozaki_slices <= 8) { ctx->cfg.ozaki_slices = cfg->ozaki_slices; ctx->oz_S = cfg->ozaki_slices; }
  return AGP_OK;
}
int32_t agp_get_config(const agp_ctx* ctx, agp_config* out) {
  if (!ctx || !out) return AGP_ERR_INVALID;
  *out = ctx->cfg;
  out->ozaki_slices = ctx->oz_S;
  out->profile_kernels = ctx->profile;
  return AGP_OK;
}
int32_t agp_last_timings(const agp_ctx* ctx, double* out, int32_t n) {
  if (!ctx || !out) return 0;
  int c = n < 8 ? n : 8;
  for (int i = 0; i < c; ++i) out[i] = ctx->timings[i];
  return c;
}
int64_t agp_launch_count(const agp_ctx*) { return agp_kernel_launches(); }

int32_t agp_gram(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, int32_t layout, const void* X, int64_t N,
                 int32_t D, const void* Z, int64_t M, const agp_noise* noise, void* K_out) {
  if (!ctx) return AGP_ERR_INVALID;
  return DISPATCH(dtype, gram_impl<float>(ctx, k, layout, X, N, D, Z, M, noise, K_out),
                  gram_impl<double>(ctx, k, layout, X, N, D, Z, M, noise, K_out));
}

int32_t agp_fit(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                int32_t layout, const void* X, int64_t N, int32_t D, const void* Y, int32_t S, void* logpdf_out,
                void* alpha_out, agp_post** post_out) {
  if (!ctx) return AGP_ERR_INVALID;
  if (post_out) *post_out = nullptr;
  if (ctx->nccl) {  // distributed context: every rank calls with the same (replicated) inputs
    return DISPATCH(dtype, fit_dist_impl<float>(ctx, k, mean, noise, layout, X, N, D, Y, S, logpdf_out, alpha_out, post_out),
                    fit_dist_impl<double>(ctx, k, mean, noise, layout, X, N, D, Y, S, logpdf_out, alpha_out, post_out));
  }
  return DISPATCH(dtype, fit_many_impl<float>(ctx, k, mean, noise, layout, X, N, D, Y, S, logpdf_out, alpha_out, post_out),
                  fit_many_impl<double>(ctx, k, mean, noise, layout, X, N, D, Y, S, logpdf_out, alpha_out, post_out));
}

int32_t agp_post_mean_var(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                          const agp_noise* noise_s, void* mean_out, void* var_out) {
  if (!p) return AGP_ERR_INVALID;
  if (p->dist_R > 1)
    return DISPATCH(p->dtype, post_mean_var_dist<float>(p, layout, Xs, M, mean_s, noise_s, mean_out, var_out),
                    post_mean_var_dist<double>(p, layout, Xs, M, mean_s, noise_s, mean_out, var_out));
  return DISPATCH(p->dtype, post_mean_var_impl<float>(p, layout, Xs, M, mean_s, noise_s, mean_out, var_out),
                  post_mean_var_impl<double>(p, layout, Xs, M, mean_s, noise_s, mean_out, var_out));
}

int32_t agp_post_mean_cov(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                          void* mean_out, void* cov_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype, post_mean_cov_impl<float>(p, layout, Xs, M, mean_s, mean_out, cov_out),
                  post_mean_cov_impl<double>(p, layout, Xs, M, mean_s, mean_out, cov_out));
}

int32_t agp_post_logpdf(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                        const agp_noise* noise_s, const void* Y, int32_t S, void* logpdf_out) {
  if (!p) return AGP_ERR_INVALID;
  if (S <= 0) { p->ctx->err = "S must be positive"; return AGP_ERR_INVALID; }
  return DISPATCH(p->dtype, post_cond_impl<float>(p, layout, Xs, M, mean_s, noise_s, Y, S, logpdf_out, nullptr, 0, nullptr),
                  post_cond_impl<double>(p, layout, Xs, M, mean_s, noise_s, Y, S, logpdf_out, nullptr, 0, nullptr));
}

int32_t agp_post_rand(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                      const agp_noise* noise_s, const void* Z, int32_t S, void* out) {
  if (!p) return AGP_ERR_INVALID;
  if (S <= 0) return AGP_OK;
  return DISPATCH(p->dtype, post_cond_impl<float>(p, layout, Xs, M, mean_s, noise_s, nullptr, 0, nullptr, Z, S, out),
                  post_cond_impl<double>(p, layout, Xs, M, mean_s, noise_s, nullptr, 0, nullptr, Z, S, out));
}

int32_t agp_post_logpdf_grad(agp_post* p, double* grad_out, void* noise_diag_out) {
  if (!p || !grad_out) return AGP_ERR_INVALID;
  return agp_post_logpdf_grad_x(p, grad_out, noise_diag_out, AGP_POINT_MAJOR, nullptr);
}

int32_t agp_post_logpdf_grad_x(agp_post* p, double* grad_out, void* noise_diag_out, int32_t layout, void* x_grad_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype, post_logpdf_grad_impl<float>(p, grad_out, noise_diag_out, layout, x_grad_out),
                  post_logpdf_grad_impl<double>(p, grad_out, noise_diag_out, layout, x_grad_out));
}

int32_t agp_post_logpdf_grad_cols(agp_post* p, const agp_mean* mean, const void* Y, int32_t S, const double* lp_bar,
                                  double* grad_out, void* noise_diag_out, void* mean_diag_out, int32_t layout,
                                  void* x_grad_out, void* y_bar_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype,
                  post_logpdf_grad_cols_impl<float>(p, mean, Y, S, lp_bar, grad_out, noise_diag_out, mean_diag_out, layout,
                                                    x_grad_out, y_bar_out),
                  post_logpdf_grad_cols_impl<double>(p, mean, Y, S, lp_bar, grad_out, noise_diag_out, mean_diag_out, layout,
                                                     x_grad_out, y_bar_out));
}

int32_t agp_post_pred_logpdf_grad(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                                  const agp_noise* noise_s, const void* Ys, int32_t S, const double* lp_bar, void* lp_out,
                                  double* grad_out, void* noise_diag_out, void* mean_diag_out, void* y_bar_out,
                                  void* x_grad_out, void* noise_s_diag_out, void* mean_s_diag_out, void* ys_bar_out,
                                  void* xs_grad_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype,
                  post_pred_logpdf_grad_impl<float>(p, layout, Xs, M, mean_s, noise_s, Ys, S, lp_bar, lp_out, grad_out,
                                                    noise_diag_out, mean_diag_out, y_bar_out, x_grad_out, noise_s_diag_out,
                                                    mean_s_diag_out, ys_bar_out, xs_grad_out),
                  post_pred_logpdf_grad_impl<double>(p, layout, Xs, M, mean_s, noise_s, Ys, S, lp_bar, lp_out, grad_out,
                                                     noise_diag_out, mean_diag_out, y_bar_out, x_grad_out, noise_s_diag_out,
                                                     mean_s_diag_out, ys_bar_out, xs_grad_out));
}

int32_t agp_post_rand_grad(agp_post* p, int32_t layout, const void* Xs, int64_t M, const agp_mean* mean_s,
                           const agp_noise* noise_s, const void* Z, int32_t S, const void* out_bar, double* grad_out,
                           void* noise_diag_out, void* mean_diag_out, void* y_bar_out, void* x_grad_out,
                           void* noise_s_diag_out, void* mean_s_diag_out, void* z_bar_out, void* xs_grad_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype,
                  post_rand_grad_impl<float>(p, layout, Xs, M, mean_s, noise_s, Z, S, out_bar, grad_out, noise_diag_out,
                                             mean_diag_out, y_bar_out, x_grad_out, noise_s_diag_out, mean_s_diag_out,
                                             z_bar_out, xs_grad_out),
                  post_rand_grad_impl<double>(p, layout, Xs, M, mean_s, noise_s, Z, S, out_bar, grad_out, noise_diag_out,
                                              mean_diag_out, y_bar_out, x_grad_out, noise_s_diag_out, mean_s_diag_out,
                                              z_bar_out, xs_grad_out));
}

int32_t agp_post_mean_var_grad(agp_post* p, int32_t layout, const void* Xs, int64_t M, const void* mean_bar,
                               const void* var_bar, double* grad_out, void* noise_diag_out, void* mean_diag_out,
                               void* y_bar_out, void* x_grad_out, void* xs_grad_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype,
                  post_mean_var_grad_impl<float>(p, layout, Xs, M, mean_bar, var_bar, grad_out, noise_diag_out,
                                                 mean_diag_out, y_bar_out, x_grad_out, xs_grad_out),
                  post_mean_var_grad_impl<double>(p, layout, Xs, M, mean_bar, var_bar, grad_out, noise_diag_out,
                                                  mean_diag_out, y_bar_out, x_grad_out, xs_grad_out));
}

int32_t agp_post_solve_lower(agp_post* p, const void* B, int64_t nrhs, void* V_out) {
  if (!p || !B || !V_out) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype, post_solve_lower_impl<float>(p, B, nrhs, V_out), post_solve_lower_impl<double>(p, B, nrhs, V_out));
}

int32_t agp_post_factor_export(agp_post* p, void* U_out) {
  if (!p || !U_out) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype, post_export_impl<float>(p, U_out), post_export_impl<double>(p, U_out));
}

int32_t agp_post_logdet(agp_post* p, double* out) {
  if (!p || !out) return AGP_ERR_INVALID;
  *out = p->logdet;
  return AGP_OK;
}
int64_t agp_post_n(const agp_post* p) { return p ? p->n : 0; }

int32_t agp_post_free(agp_post* p) {
  if (!p) return AGP_OK;
  cudaSetDevice(p->ctx->device);
  cudaStream_t s = p->ctx->stream;
  if (p->L) cudaFreeAsync(p->L, s);
  if (p->Dinv) cudaFreeAsync(p->Dinv, s);
  if (p->Xt) cudaFreeAsync(p->Xt, s);
  if (p->alpha) cudaFreeAsync(p->alpha, s);
  if (p->ard) cudaFreeAsync(p->ard, s);
  if (p->delta) cudaFreeAsync(p->delta, s);
  if (p->valid) cudaFreeAsync(p->valid, s);
  if (p->Lloc) cudaFreeAsync(p->Lloc, s);
  if (p->Dinv_loc) cudaFreeAsync(p->Dinv_loc, s);
  comp_free(p->comp, s);
  delete p;
  return AGP_OK;
}

int64_t agp_post_grad_len(const agp_post* p) {
  if (!p) return 0;
  return p->comp ? p->comp->grad_len : 5 + (int64_t)p->D;
}

int32_t agp_rand(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                 int32_t layout, const void* X, int64_t N, int32_t D, const void* Z, int32_t S, void* out) {
  if (!ctx) return AGP_ERR_INVALID;
  return DISPATCH(dtype, rand_impl<float>(ctx, k, mean, noise, layout, X, N, D, Z, S, out),
                  rand_impl<double>(ctx, k, mean, noise, layout, X, N, D, Z, S, out));
}

int32_t agp_rand_grad(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                      int32_t layout, const void* X, int64_t N, int32_t D, const void* Z, int32_t S, const void* out_bar,
                      double* grad_out, void* noise_diag_out, void* mean_diag_out, void* x_grad_out, void* z_bar_out) {
  if (!ctx) return AGP_ERR_INVALID;
  int rc = rand_grad_check(ctx, layout, X, Z, S, out_bar);
  if (rc) return rc;
  return DISPATCH(dtype, rand_grad_f32(ctx, k, mean, noise, layout, X, N, D, Z, S, out_bar, grad_out, noise_diag_out,
                                       mean_diag_out, x_grad_out, z_bar_out),
                  rand_grad_f64(ctx, k, mean, noise, layout, X, N, D, Z, S, out_bar, grad_out, noise_diag_out,
                                mean_diag_out, x_grad_out, z_bar_out));
}

int32_t agp_debug_ozaki_syrk(agp_ctx* ctx, void* C_dev, int64_t ldc, const void* P_dev, int64_t lda, int64_t M, int64_t N,
                             int32_t K, int32_t S, int32_t lower_only) {
  if (!ctx || !C_dev || !P_dev) return AGP_ERR_INVALID;
  // the N columns pair with panel rows 0 .. N-1, so they must be among the M rows that are sliced
  if (M <= 0 || N <= 0 || N > M || ldc < M) { ctx->err = "ozaki syrk: need 0 < N <= M <= ldc"; return AGP_ERR_INVALID; }
  if (S < 5 || S > 8) { ctx->err = "ozaki syrk: fp64 C takes 5..8 slices"; return AGP_ERR_UNSUPPORTED; }
  cudaSetDevice(ctx->device);
  OzakiWs ws;
  int rc = ozaki_ws_create(&ws, M, K, S, ctx->stream);
  if (rc) { ctx->err = "ozaki_ws_create failed (code " + std::to_string(rc) + ")"; return rc == 1 ? AGP_ERR_INVALID : AGP_ERR_CUDA; }
  ozaki_prepare(ws, (const double*)P_dev, lda, M, ctx->stream);
  const int urc = ozaki_syrk(ws, (double*)C_dev, ldc, M, N, lower_only, 0, 0, 0, 0, ctx->stream);
  ozaki_ws_destroy(&ws, ctx->stream);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { ctx->err = std::string("ozaki syrk: ") + cudaGetErrorString(e); return AGP_ERR_CUDA; }
  if (urc) { ctx->err = "ozaki syrk: slice count or strip table not supported"; return AGP_ERR_UNSUPPORTED; }
  return AGP_OK;
}

// general product on the int8-slice path: C (M x N, fp32 or fp64) += sign * A B', A = M x K, B = N x K (B_dev == NULL: B = A,
// lower tiles only).  Each operand is fp32 or fp64, row-contiguous (element (r, k) at [r + k*ld]) or k-major ([k + r*ld]).
// Both operands are sliced into one workspace (A rows first, B rows from the next multiple of 128).
int32_t agp_debug_ozaki_gemm(agp_ctx* ctx, void* C_dev, int32_t c_is_float, int64_t ldc, const void* A_dev, int32_t a_is_float,
                             int32_t a_kmajor, int64_t lda, int64_t M, const void* B_dev, int32_t b_is_float, int32_t b_kmajor,
                             int64_t ldb, int64_t N, int32_t K, int32_t S, double sign) {
  if (!ctx || !C_dev || !A_dev) return AGP_ERR_INVALID;
  // without B the N columns pair with rows 0 .. N-1 of A, so they must be among its M sliced rows
  if (M <= 0 || N <= 0 || ldc < M || (!B_dev && N > M)) { ctx->err = "ozaki gemm: need 0 < M <= ldc, 0 < N (N <= M without B)"; return AGP_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  const int64_t m_pad = (M + 127) / 128 * 128, n_rows = B_dev ? (N + 127) / 128 * 128 : 0;
  OzakiWs ws;
  int rc = ozaki_ws_create(&ws, m_pad + n_rows, K, S, ctx->stream);
  if (rc) { ctx->err = "ozaki_ws_create failed (code " + std::to_string(rc) + ")"; return rc == 1 ? AGP_ERR_INVALID : AGP_ERR_CUDA; }
  ozaki_prepare_ex(ws, A_dev, a_is_float, a_kmajor, lda, M, 0, ctx->stream);
  if (B_dev) ozaki_prepare_ex(ws, B_dev, b_is_float, b_kmajor, ldb, N, m_pad, ctx->stream);
  const int urc = ozaki_update_ex(ws, C_dev, c_is_float, ldc, M, N, B_dev ? 1 : 0, sign, 0, 0, B_dev ? m_pad : 0, 0, ctx->stream);
  ozaki_ws_destroy(&ws, ctx->stream);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (urc) { ctx->err = "ozaki_update_ex: unsupported shape / slice count (N % 128, S)"; return AGP_ERR_UNSUPPORTED; }
  if (e != cudaSuccess) { ctx->err = std::string("ozaki gemm: ") + cudaGetErrorString(e); return AGP_ERR_CUDA; }
  return AGP_OK;
}

// block-cyclic column map of the distributed trailing update on ONE device: P has m_panel rows; row r of C pairs with
// panel row r + a_off, local column n with panel row (n / b_tile_width) * b_tile_stride + n % b_tile_width + b_off.
// This drives the strip-table enumeration of the persistent kernel exactly as fit_dist_impl does.
int32_t agp_debug_ozaki_syrk_map(agp_ctx* ctx, void* C_dev, int64_t ldc, const void* P_dev, int64_t lda, int64_t m_panel,
                                 int64_t M, int64_t N, int32_t K, int32_t S, int64_t b_tile_stride, int64_t b_tile_width,
                                 int64_t b_off, int64_t a_off) {
  if (!ctx || !C_dev || !P_dev) return AGP_ERR_INVALID;
  if (N % 128 != 0 || N < 128 || M <= 0 || m_panel <= 0) { ctx->err = "N must be a positive multiple of 128"; return AGP_ERR_INVALID; }
  // rows and columns address the sliced panel in whole 128-row blocks: offsets and the column map must stay inside it
  const int64_t bw = b_tile_width ? b_tile_width : 128;
  const int64_t last_col_row = (b_tile_stride ? ((N - 1) / bw) * b_tile_stride + (N - 1) % bw : N - 1) + b_off;
  if (a_off < 0 || b_off < 0 || a_off % 128 || b_off % 128 || b_tile_stride % 128 || bw % 128 || ldc < M ||
      M + a_off > m_panel || last_col_row >= m_panel) {
    ctx->err = "ozaki syrk (map): rows or columns outside the panel (offsets, stride and width in multiples of 128)";
    return AGP_ERR_INVALID;
  }
  if (S < 5 || S > 8) { ctx->err = "ozaki syrk (map): fp64 C takes 5..8 slices"; return AGP_ERR_UNSUPPORTED; }
  cudaSetDevice(ctx->device);
  OzakiWs ws;
  int rc = ozaki_ws_create(&ws, m_panel, K, S, ctx->stream);
  if (rc) { ctx->err = "ozaki_ws_create failed (code " + std::to_string(rc) + ")"; return rc == 1 ? AGP_ERR_INVALID : AGP_ERR_CUDA; }
  ozaki_prepare(ws, (const double*)P_dev, lda, m_panel, ctx->stream);
  const int urc = ozaki_syrk(ws, (double*)C_dev, ldc, M, N, 1, b_tile_stride, b_tile_width, b_off, a_off, ctx->stream);
  ozaki_ws_destroy(&ws, ctx->stream);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { ctx->err = std::string("ozaki syrk (map): ") + cudaGetErrorString(e); return AGP_ERR_CUDA; }
  if (urc) { ctx->err = "ozaki syrk (map): strip table not supported"; return AGP_ERR_UNSUPPORTED; }
  return AGP_OK;
}

int32_t agp_debug_ozaki8(agp_ctx* ctx, void* C_dev, int64_t ldc, const void* A_dev, int32_t a_kmajor, int64_t lda,
                         int64_t m_panel, const void* B_dev, int32_t b_kmajor, int64_t ldb, int64_t M, int64_t N, int32_t K,
                         double sign, int64_t b_tile_stride, int64_t b_tile_width, int64_t b_off, int64_t a_off) {
  if (!ctx || !C_dev || !A_dev) return AGP_ERR_INVALID;
  if (N % 128 != 0 || N < 128 || M <= 0 || ldc < M) { ctx->err = "ozaki8: need 0 < M <= ldc, N a positive multiple of 128"; return AGP_ERR_INVALID; }
  const int64_t m_pad = (M + 127) / 128 * 128;
  if (B_dev) {
    if (m_panel || b_tile_stride || b_tile_width || b_off || a_off) {
      ctx->err = "ozaki8: a product with B takes no panel, column map or offsets";
      return AGP_ERR_INVALID;
    }
  } else {
    // rows and columns address the sliced panel in whole 128-row blocks: offsets and the column map must stay inside it
    const int64_t bw = b_tile_width ? b_tile_width : 128;
    const int64_t last_col_row = (b_tile_stride ? ((N - 1) / bw) * b_tile_stride + (N - 1) % bw : N - 1) + b_off;
    if (m_panel <= 0 || a_off < 0 || b_off < 0 || a_off % 128 || b_off % 128 || b_tile_stride % 128 || bw % 128 ||
        M + a_off > m_panel || last_col_row >= m_panel) {
      ctx->err = "ozaki8: rows or columns outside the panel (offsets, stride and width in multiples of 128)";
      return AGP_ERR_INVALID;
    }
  }
  cudaSetDevice(ctx->device);
  OzakiWs ws;
  int rc = ozaki_ws_create(&ws, B_dev ? m_pad + N : m_panel, K, 6, ctx->stream, 8);
  if (rc) { ctx->err = "ozaki_ws_create failed (code " + std::to_string(rc) + ")"; return rc == 1 ? AGP_ERR_INVALID : AGP_ERR_CUDA; }
  ozaki_prepare_ex(ws, A_dev, 0, a_kmajor, lda, B_dev ? M : m_panel, 0, ctx->stream);
  if (B_dev) ozaki_prepare_ex(ws, B_dev, 0, b_kmajor, ldb, N, m_pad, ctx->stream);
  const int urc = ozaki_update_ex(ws, C_dev, 0, ldc, M, N, B_dev ? 1 : 0, sign, b_tile_stride, b_tile_width,
                                  B_dev ? m_pad : b_off, a_off, ctx->stream);
  ozaki_ws_destroy(&ws, ctx->stream);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { ctx->err = std::string("ozaki8: ") + cudaGetErrorString(e); return AGP_ERR_CUDA; }
  if (urc) { ctx->err = "ozaki8: K above 16384 or strip table not supported"; return AGP_ERR_UNSUPPORTED; }
  return AGP_OK;
}

int32_t agp_debug_gemm(agp_ctx* ctx, int32_t dtype, const void* A_dev, int32_t a_kmajor, int64_t lda, const void* B_dev,
                       int32_t b_kmajor, int64_t ldb, void* C_dev, int64_t ldc, int64_t M, int64_t N, int64_t K,
                       int32_t alpha_neg, int32_t beta_one, int32_t lower_only, int32_t trmm_lower, int64_t b_tile_stride,
                       int64_t b_tile_width, int64_t b_off) {
  if (!ctx || !A_dev || !B_dev || !C_dev) return AGP_ERR_INVALID;
  if (dtype != AGP_F32 && dtype != AGP_F64) { ctx->err = "gemm: dtype must be AGP_F32 or AGP_F64"; return AGP_ERR_INVALID; }
  cudaSetDevice(ctx->device);
  GemmArgs g{};
  g.A = A_dev; g.lda = lda; g.a_kmajor = a_kmajor != 0;
  g.B = B_dev; g.ldb = ldb; g.b_kmajor = b_kmajor != 0;
  g.C = C_dev; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
  g.alpha_neg = alpha_neg != 0; g.beta_one = beta_one != 0; g.lower_only = lower_only != 0; g.trmm_lower = trmm_lower != 0;
  g.b_tile_stride = b_tile_stride; g.b_tile_width = b_tile_width; g.b_off = b_off;
  const int rc = dtype == AGP_F64 ? launch_gemm<double>(g, ctx->stream) : launch_gemm<float>(g, ctx->stream);
  if (rc) { ctx->err = "gemm: the operands break the tile GEMM's contract (csrc/kernels.h)"; return AGP_ERR_INVALID; }
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { ctx->err = std::string("gemm: ") + cudaGetErrorString(e); return AGP_ERR_CUDA; }
  return AGP_OK;
}

int32_t agp_debug_panel(agp_ctx* ctx, int32_t dtype, int32_t route, void* A_dev, int64_t lda, int64_t rows_below,
                        int32_t blk, void* Dinv_dev, double* logdet_dev, int32_t* info_dev) {
  if (!ctx || !A_dev || !Dinv_dev || !logdet_dev || !info_dev) return AGP_ERR_INVALID;
  if (dtype != AGP_F32 && dtype != AGP_F64) { ctx->err = "panel: dtype must be AGP_F32 or AGP_F64"; return AGP_ERR_INVALID; }
  if (route != AGP_PANEL_FUSED && (dtype != AGP_F64 || (route != AGP_PANEL_SPLIT_SUBST && route != AGP_PANEL_SPLIT_GEMM))) {
    ctx->err = "panel: the split routes are fp64 only";
    return AGP_ERR_INVALID;
  }
  // the panel GEMM reads A21 and Dinv in 16-byte loads (the GemmArgs contract)
  const int64_t vec = dtype == AGP_F64 ? 2 : 4;
  if (rows_below < 0 || blk < 0 || lda < TILE + rows_below || lda % vec || ((uintptr_t)A_dev & 15) ||
      ((uintptr_t)Dinv_dev & 15)) {
    ctx->err = "panel: need 0 <= rows_below <= lda - 128, blk >= 0, lda and the pointers aligned to 16 bytes";
    return AGP_ERR_INVALID;
  }
  if (dtype == AGP_F32 && rows_below % 4) {  // the fp32 panel GEMM stores float4 row quads (M % 4 == 0)
    ctx->err = "panel: an fp32 panel needs rows_below % 4 == 0";
    return AGP_ERR_INVALID;
  }
  cudaSetDevice(ctx->device);
  if (dtype == AGP_F64)
    panel_block<double>(ctx, route, (double*)A_dev, lda, rows_below, (double*)Dinv_dev, logdet_dev, blk, info_dev, ctx->stream);
  else
    panel_block<float>(ctx, route, (float*)A_dev, lda, rows_below, (float*)Dinv_dev, logdet_dev, blk, info_dev, ctx->stream);
  join_inverses(ctx);
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { ctx->err = std::string("panel: ") + cudaGetErrorString(e); return AGP_ERR_CUDA; }
  return AGP_OK;
}

int32_t agp_bc_owner(int32_t ti, int32_t tj, int32_t P, int32_t Q) { return (ti % P) * Q + (tj % Q); }
int64_t agp_bc_local_tiles(int32_t nt, int32_t rank, int32_t P, int32_t Q) {
  int64_t c = 0;
  for (int i = 0; i < nt; ++i)
    for (int j = 0; j <= i; ++j)
      if (agp_bc_owner(i, j, P, Q) == rank) ++c;
  return c;
}

// ---- multi-GPU entry points are provided by dist.cu ------------------------------------------------
int32_t agp_post_extend(agp_post* p, int32_t layout, const void* X2, int64_t N2, const void* y2, const agp_mean* mean2,
                        const agp_noise* noise2, void* alpha_out, agp_post** post_out) {
  if (!p) return AGP_ERR_INVALID;
  if (post_out) *post_out = nullptr;
  return DISPATCH(p->dtype, post_extend_impl<float>(p, layout, X2, N2, y2, mean2, noise2, alpha_out, post_out),
                  post_extend_impl<double>(p, layout, X2, N2, y2, mean2, noise2, alpha_out, post_out));
}
int32_t agp_vfe_elbo(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                     int32_t layout, const void* X, int64_t N, int32_t D, const void* Zind, int64_t M,
                     const agp_noise* jitter, const void* y, void* elbo_out, void* dtc_out) {
  if (!ctx) return AGP_ERR_INVALID;
  return DISPATCH(dtype, vfe_core<float>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, elbo_out, dtc_out, nullptr),
                  vfe_core<double>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, elbo_out, dtc_out, nullptr));
}
int32_t agp_vfe_elbo_grad_x(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                            int32_t layout, const void* X, int64_t N, int32_t D, const void* Zind, int64_t M,
                            const agp_noise* jitter, const void* y, int32_t objective, void* value_out, double* grad_out,
                            void* noise_diag_out, void* mean_diag_out, void* z_grad_out, void* x_grad_out) {
  if (!ctx) return AGP_ERR_INVALID;
  int rc = vfe_grad_check(ctx, k, layout, objective);
  if (rc) return rc;
  return DISPATCH(dtype,
                  vfe_grad_f32(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, objective, value_out, grad_out,
                               noise_diag_out, mean_diag_out, z_grad_out, x_grad_out),
                  vfe_grad_impl<double>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, objective, value_out,
                                        grad_out, noise_diag_out, mean_diag_out, z_grad_out, x_grad_out));
}
int32_t agp_vfe_elbo_grad(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                          int32_t layout, const void* X, int64_t N, int32_t D, const void* Zind, int64_t M,
                          const agp_noise* jitter, const void* y, int32_t objective, void* value_out, double* grad_out,
                          void* noise_diag_out, void* mean_diag_out, void* z_grad_out) {
  return agp_vfe_elbo_grad_x(ctx, dtype, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, objective, value_out, grad_out,
                             noise_diag_out, mean_diag_out, z_grad_out, nullptr);
}
int32_t agp_vfe_fit(agp_ctx* ctx, int32_t dtype, const agp_kernel* k, const agp_mean* mean, const agp_noise* noise,
                    int32_t layout, const void* X, int64_t N, int32_t D, const void* Zind, int64_t M,
                    const agp_noise* jitter, const void* y, agp_vfe_post** out) {
  if (!ctx || !out) return AGP_ERR_INVALID;
  *out = nullptr;
  return DISPATCH(dtype, vfe_core<float>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, nullptr, nullptr, out),
                  vfe_core<double>(ctx, k, mean, noise, layout, X, N, D, Zind, M, jitter, y, nullptr, nullptr, out));
}
int32_t agp_vfe_mean_var(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t Ms, void* mean_out, void* var_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype, vfe_mean_var_impl<float>(p, layout, Xs, Ms, mean_out, var_out),
                  vfe_mean_var_impl<double>(p, layout, Xs, Ms, mean_out, var_out));
}
int32_t agp_vfe_mean_cov(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t M, void* mean_out, void* cov_out) {
  if (!p) return AGP_ERR_INVALID;
  return DISPATCH(p->dtype, vfe_cond_impl<float>(p, layout, Xs, M, nullptr, mean_out, cov_out, nullptr, 0, nullptr, nullptr, 0, nullptr),
                  vfe_cond_impl<double>(p, layout, Xs, M, nullptr, mean_out, cov_out, nullptr, 0, nullptr, nullptr, 0, nullptr));
}
int32_t agp_vfe_post_logpdf(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t M, const agp_noise* noise_s,
                            const void* Y, int32_t S, void* logpdf_out) {
  if (!p) return AGP_ERR_INVALID;
  if (S <= 0) { p->ctx->err = "S must be positive"; return AGP_ERR_INVALID; }
  return DISPATCH(p->dtype, vfe_cond_impl<float>(p, layout, Xs, M, noise_s, nullptr, nullptr, Y, S, logpdf_out, nullptr, 0, nullptr),
                  vfe_cond_impl<double>(p, layout, Xs, M, noise_s, nullptr, nullptr, Y, S, logpdf_out, nullptr, 0, nullptr));
}
int32_t agp_vfe_post_rand(agp_vfe_post* p, int32_t layout, const void* Xs, int64_t M, const agp_noise* noise_s,
                          const void* Z, int32_t S, void* out) {
  if (!p) return AGP_ERR_INVALID;
  if (S <= 0) return AGP_OK;
  return DISPATCH(p->dtype, vfe_cond_impl<float>(p, layout, Xs, M, noise_s, nullptr, nullptr, nullptr, 0, nullptr, Z, S, out),
                  vfe_cond_impl<double>(p, layout, Xs, M, noise_s, nullptr, nullptr, nullptr, 0, nullptr, Z, S, out));
}
int32_t agp_vfe_post_free(agp_vfe_post* p) {
  if (!p) return AGP_OK;
  cudaSetDevice(p->ctx->device);
  cudaStream_t s = p->ctx->stream;
  void* ptrs[] = {p->U, p->Udinv, p->Lam, p->Ldinv, p->Zt, p->m_e, p->ard};
  for (void* q : ptrs) if (q) cudaFreeAsync(q, s);
  delete p;
  return AGP_OK;
}
int32_t agp_nccl_unique_id(void* out128) {
  if (!out128) return AGP_ERR_INVALID;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  if (ncclGetUniqueId(&id) != ncclSuccess) return AGP_ERR_NCCL;
  memcpy(out128, &id, 128);
  return AGP_OK;
}
int32_t agp_init_dist(agp_ctx** out, int32_t device, int32_t rank, int32_t nranks, int32_t grid_p, int32_t grid_q,
                      const void* id128, const agp_config* cfg) {
  if (!out || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return AGP_ERR_INVALID;
  if (grid_p != 1 || grid_q != nranks) return AGP_ERR_UNSUPPORTED;  // 1 x Q block-column-cyclic grid in this build
  int32_t rc = agp_init(out, device, cfg);
  if (rc != AGP_OK) return rc;
  agp_ctx* ctx = *out;
  ctx->rank = rank; ctx->nranks = nranks; ctx->grid_p = grid_p; ctx->grid_q = grid_q;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  // the panel broadcasts run beside the persistent trailing-update kernel, which leaves a few SMs free: keep NCCL's
  // kernels within that reserve
  ncclConfig_t ncfg = NCCL_CONFIG_INITIALIZER;
  ncfg.maxCTAs = env_int("AGP_NCCL_MAX_CTAS", 16);
  if (ncclCommInitRankConfig(&ctx->nccl, nranks, id, rank, &ncfg) != ncclSuccess) {
    agp_destroy(ctx);
    *out = nullptr;
    return AGP_ERR_NCCL;
  }
  return AGP_OK;
}

}  // extern "C"

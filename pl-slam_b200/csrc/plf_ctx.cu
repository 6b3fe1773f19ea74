// Context lifetime, error reporting, scratch memory.  Host-side plumbing only; no kernels here.
#include <stdarg.h>

#include "plf_internal.h"
#include <cstdlib>
#include <cstdio>
#include <cstring>

static thread_local std::string g_create_err;

plf_status plf_fail(plf_ctx* ctx, plf_status code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx)
    ctx->err = buf;
  else
    g_create_err = buf;
  return code;
}

size_t DevBufList::bytes() const {
  size_t n = 0;
  for (const Entry& e : entries) n += e.bytes;
  return n;
}

plf_status DevBufList::alloc(plf_ctx* ctx, const char* owner) {
  for (const Entry& e : entries) {
    const cudaError_t err = cudaMalloc(e.slot, e.bytes + 64);
    if (err != cudaSuccess) {
      *e.slot = nullptr;
      return plf_fail(ctx, PLF_ERR_CUDA, "%s: cudaMalloc(%zu): %s", owner, e.bytes, cudaGetErrorString(err));
    }
  }
  return PLF_OK;
}

void DevBufList::release() {
  for (const Entry& e : entries) {
    cudaFree(*e.slot);
    *e.slot = nullptr;
  }
}

void* plf_scratch(plf_ctx* ctx, int slot, size_t bytes) {
  DevBuf& b = ctx->scratch[slot];
  if (b.bytes >= bytes && b.p) return b.p;
  if (b.p) {
    cudaStreamSynchronize(ctx->stream);
    cudaFree(b.p);
    b.p = nullptr;
    b.bytes = 0;
  }
  size_t want = bytes < 4096 ? 4096 : bytes;
  want = (want + 255) & ~size_t(255);
  cudaError_t e = cudaMalloc(&b.p, want + 64);  // + slack for plf_load4 (see plf_image_span)
  if (e != cudaSuccess) {
    plf_fail(ctx, PLF_ERR_CUDA, "cudaMalloc(%zu) scratch slot %d: %s", want, slot,
             cudaGetErrorString(e));
    b.p = nullptr;
    return nullptr;
  }
  b.bytes = want;
  return b.p;
}

void* plf_pinned(plf_ctx* ctx, size_t bytes) {
  if (ctx->pinned_bytes >= bytes && ctx->pinned) return ctx->pinned;
  if (ctx->pinned) {
    cudaStreamSynchronize(ctx->stream);
    cudaFreeHost(ctx->pinned);
    ctx->pinned = nullptr;
    ctx->pinned_bytes = 0;
  }
  size_t want = bytes < (1 << 20) ? (1 << 20) : bytes;
  cudaError_t e = cudaHostAlloc(&ctx->pinned, want, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    plf_fail(ctx, PLF_ERR_CUDA, "cudaHostAlloc(%zu): %s", want, cudaGetErrorString(e));
    ctx->pinned = nullptr;
    return nullptr;
  }
  ctx->pinned_bytes = want;
  return ctx->pinned;
}

void plf_mark(plf_ctx* ctx, const char* name) {
  if (!ctx->profile) return;
  if (ctx->prof_used == ctx->prof_ev.size()) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) return;
    ctx->prof_ev.push_back(e);
    ctx->prof_names.emplace_back();
  }
  ctx->prof_names[ctx->prof_used] = name;
  cudaEventRecord(ctx->prof_ev[ctx->prof_used], ctx->cur);
  ctx->prof_used++;
}

extern "C" {

plf_status plf_profile_enable(plf_ctx* ctx, int on) {
  if (!ctx) return PLF_ERR_INVALID;
  ctx->profile = on != 0;
  ctx->profile_piped = on == 2;
  ctx->prof_used = 0;
  return PLF_OK;
}

// After a plf_batch_run with profiling on: per-stage device time (ms) between consecutive marks.
// names_buf receives the stage names separated by ';'.  Resets the mark list.
plf_status plf_profile_read(plf_ctx* ctx, char* names_buf, int buf_len, float* ms, int cap, int* n_out) {
  if (!ctx || !n_out) return PLF_ERR_INVALID;
  if (ctx->profile_piped) PLF_CUDA(ctx, cudaDeviceSynchronize());
  else PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int n = 0;
  std::string names;
  for (size_t i = 1; i < ctx->prof_used; ++i) {
    if (n < cap && ms) {
      float t = 0;
      cudaEventElapsedTime(&t, ctx->prof_ev[i - 1], ctx->prof_ev[i]);
      ms[n] = t;
    }
    names += ctx->prof_names[i];
    names += ';';
    ++n;
  }
  if (names_buf && buf_len > 0) {
    strncpy(names_buf, names.c_str(), buf_len - 1);
    names_buf[buf_len - 1] = 0;
  }
  *n_out = n;
  ctx->prof_used = 0;
  return PLF_OK;
}

int plf_abi_version(void) { return PLF_ABI_VERSION; }

const char* plf_last_error(const plf_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_create_err.c_str();
}

// Defaults = config/config/config_euroc.yaml:9-77 of the reference.
void plf_default_params(plf_params* p) {
  memset(p, 0, sizeof *p);
  p->has_points = 1;
  p->has_lines = 1;
  p->best_lr_matches = 1;
  p->max_dist_epip = 1.0f;
  p->min_disp = 1.0f;
  p->min_ratio_12_p = 0.9f;
  p->line_sim_th = 0.75f;
  p->stereo_overlap_th = 0.75f;
  p->f2f_overlap_th = 0.75f;
  p->min_line_length = 0.025f;
  p->line_horiz_th = 0.1f;
  p->min_ratio_12_l = 0.9f;
  p->ls_min_disp_ratio = 0.7f;
  p->homog_th = 1e-7;
  p->min_features = 10;
  p->max_iters = 5;
  p->max_iters_ref = 10;
  p->min_error = 1e-7;
  p->min_error_change = 1e-7;
  p->inlier_k = 4.0;
  p->orb_nfeatures = 800;
  p->orb_scale_factor = 1.2f;
  p->orb_nlevels = 4;
  p->orb_edge_th = 19;
  p->orb_wta_k = 2;
  p->orb_score = 1;
  p->orb_patch_size = 31;
  p->orb_fast_th = 20;
  p->lsd_nfeatures = 300;
  p->lsd_refine = 0;
  p->lsd_scale = 1.2;
  p->lsd_sigma_scale = 0.6;
  p->lsd_quant = 2.0;
  p->lsd_ang_th = 22.5;
  p->lsd_log_eps = 1.0;
  p->lsd_density_th = 0.6;
  p->lsd_n_bins = 1024;
  p->matching_strategy = 0;
  p->matching_s_ws = 10;
  p->matching_f2f_ws = 3;
  p->min_pt_matches = 10;
  p->min_ls_matches = 6;
}

void plf_default_limits(plf_limits* l) {
  l->max_batch = 8;
  l->max_keypoints = 4096;
  l->max_segments = 8192;
  l->max_lines = 1024;
}

void plf_destroy(plf_ctx* ctx);

plf_status plf_create(const plf_params* params, const plf_camera* cam, const plf_limits* limits,
                      int device, plf_ctx** out) {
  if (!out) return plf_fail(nullptr, PLF_ERR_INVALID, "plf_create: out is NULL");
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return plf_fail(nullptr, PLF_ERR_NO_DEVICE,
                    "plf_create: no CUDA device (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
  if (device < 0 || device >= ndev)
    return plf_fail(nullptr, PLF_ERR_INVALID, "plf_create: device %d out of range [0,%d)", device,
                    ndev);
  e = cudaSetDevice(device);
  if (e != cudaSuccess)
    return plf_fail(nullptr, PLF_ERR_NO_DEVICE, "cudaSetDevice(%d): %s", device,
                    cudaGetErrorString(e));
  plf_ctx* ctx = new plf_ctx();
  ctx->device = device;
  if (params)
    ctx->params = *params;
  else
    plf_default_params(&ctx->params);
  if (cam)
    ctx->cam = *cam;
  else {
    plf_camera c = {1242, 375, 718.856, 718.856, 607.1928, 185.2157, 0.537165719};
    ctx->cam = c;
  }
  if (limits)
    ctx->limits = *limits;
  else
    plf_default_limits(&ctx->limits);
  if (ctx->cam.width <= 0 || ctx->cam.height <= 0 || ctx->limits.max_batch <= 0) {
    delete ctx;
    return plf_fail(nullptr, PLF_ERR_INVALID, "plf_create: bad camera size or max_batch");
  }
  if (!ctx->params.has_points && !ctx->params.has_lines) {
    delete ctx;
    return plf_fail(nullptr, PLF_ERR_INVALID, "plf_create: has_points and has_lines are both 0; a front-end needs one of them");
  }
  plf_configure_lsd();
  cudaGetLastError();
  e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    delete ctx;
    return plf_fail(nullptr, PLF_ERR_NO_DEVICE, "cudaStreamCreate: %s", cudaGetErrorString(e));
  }
  ctx->cur = ctx->stream;
  bool ok = true;
  // aux[1] carries the LSD chain of the batched pipeline, the longest dependent chain of a step.  PLF_G_PRIORITY=1 gives it the
  // highest stream priority (its CTAs are dispatched ahead of the pending CTAs of the ORB / match streams).  Measured: no gain -
  // the chain is slowed by sharing issue slots with the co-resident kernels, not by waiting for CTA slots (DESIGN.md 5) - so
  // equal priorities stay the default.
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  const char* gp = getenv("PLF_G_PRIORITY");
  const bool g_high = gp && gp[0] == '1';
  for (int i = 0; i < 3 && ok; ++i)
    ok = cudaStreamCreateWithPriority(&ctx->aux[i], cudaStreamNonBlocking, (i == 1 && g_high) ? prio_hi : prio_lo) == cudaSuccess;
  if (!ok) {
    plf_destroy(ctx);
    return plf_fail(nullptr, PLF_ERR_NO_DEVICE, "plf_create: could not create auxiliary streams/events");
  }
  *out = ctx;
  return PLF_OK;
}

// subsystem destructors (defined in their own translation units)
void plf_orb_free(plf_ctx* ctx);
void plf_lsd_free(plf_ctx* ctx);
void plf_lbd_free(plf_ctx* ctx);
void plf_pipe_free(plf_ctx* ctx);

void plf_destroy(plf_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  plf_pipe_free(ctx);
  plf_orb_free(ctx);
  plf_lsd_free(ctx);
  plf_lbd_free(ctx);
  for (auto& b : ctx->scratch)
    if (b.p) cudaFree(b.p);
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  for (auto e : ctx->prof_ev) cudaEventDestroy(e);
  for (int i = 0; i < 3; ++i)
    if (ctx->aux[i]) { cudaStreamSynchronize(ctx->aux[i]); cudaStreamDestroy(ctx->aux[i]); }
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}

long long plf_launch_count(const plf_ctx* ctx) { return ctx ? ctx->launches : 0; }
void* plf_stream(const plf_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

plf_status plf_sync(plf_ctx* ctx) {
  if (!ctx) return PLF_ERR_INVALID;
  PLF_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PLF_OK;
}

}  // extern "C"

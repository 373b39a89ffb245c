// Engine-level C-ABI: the reference's seams (SURVEY.md 8b) as single calls over borrowed programs and
// their fixed I/O slots.  Pure orchestration: async copies into / out of the slots, one graph replay (or
// eager run) and the K6 update; no kernels of its own except the timestep fill.
//
// UNet lanes: the latent batch is split into n_lanes independent sub-batches, each with its own step program and
// workspace; the step graph holds the lanes as parallel branches (fork / join through captured events), so the
// latency-bound deep levels of one lane overlap with the other lanes' kernels.
#include <string.h>

#include <new>

#include "common.cuh"

struct aldm_engine {
  aldm_engine_desc d;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  cudaStream_t side[ALDM_MAX_LANES] = {};
  cudaEvent_t fork = nullptr;
  cudaEvent_t join[ALDM_MAX_LANES] = {};
};

namespace aldm {

__global__ void fill_i64_kernel(long long* p, int n, long long v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

static int copy_async(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  if (bytes == 0 || dst == src) return ALDM_OK;
  ALDM_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
  return ALDM_OK;
}

static int run_lanes_eager(aldm_engine* e, cudaStream_t st) {
  for (int l = 0; l < e->d.n_lanes; ++l) {
    int rc = aldm_program_run(e->d.lane[l].step, st);
    if (rc) return rc;
  }
  return ALDM_OK;
}

// All lanes as parallel branches of one graph: lane 0 on the capturing stream, lane l > 0 on side stream l.
static int capture_lanes(aldm_engine* e) {
  const int n = e->d.n_lanes;
  cudaStream_t cs;
  ALDM_CHECK_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
  if (!e->fork) ALDM_CHECK_CUDA(cudaEventCreateWithFlags(&e->fork, cudaEventDisableTiming));
  for (int l = 1; l < n; ++l) {
    if (!e->side[l]) ALDM_CHECK_CUDA(cudaStreamCreateWithFlags(&e->side[l], cudaStreamNonBlocking));
    if (!e->join[l]) ALDM_CHECK_CUDA(cudaEventCreateWithFlags(&e->join[l], cudaEventDisableTiming));
  }
  ALDM_CHECK_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
  int rc = ALDM_OK;
  cudaError_t ce = cudaEventRecord(e->fork, cs);
  for (int l = 1; l < n && rc == ALDM_OK && ce == cudaSuccess; ++l) {
    ce = cudaStreamWaitEvent(e->side[l], e->fork, 0);
    if (ce == cudaSuccess) rc = aldm_program_run(e->d.lane[l].step, e->side[l]);
    if (ce == cudaSuccess && rc == ALDM_OK) ce = cudaEventRecord(e->join[l], e->side[l]);
  }
  if (rc == ALDM_OK && ce == cudaSuccess) rc = aldm_program_run(e->d.lane[0].step, cs);
  for (int l = 1; l < n && rc == ALDM_OK && ce == cudaSuccess; ++l) ce = cudaStreamWaitEvent(cs, e->join[l], 0);
  cudaGraph_t g = nullptr;
  const cudaError_t ee = cudaStreamEndCapture(cs, &g);
  cudaStreamDestroy(cs);
  if (rc != ALDM_OK) { if (g) cudaGraphDestroy(g); return rc; }
  if (ce != cudaSuccess || ee != cudaSuccess) {
    if (g) cudaGraphDestroy(g);
    set_error("engine: lane graph capture failed: %s", cudaGetErrorString(ce != cudaSuccess ? ce : ee));
    return ALDM_E_CUDA;
  }
  e->graph = g;
  ALDM_CHECK_CUDA(cudaGraphInstantiate(&e->exec, e->graph, 0));
  return ALDM_OK;
}

static int run_unet(aldm_engine* e, const float* x, int64_t t, cudaStream_t st) {
  const aldm_engine_desc& d = e->d;
  const int Bl = d.B / d.n_lanes;
  for (int l = 0; l < d.n_lanes; ++l) {
    const aldm_unet_lane& ln = d.lane[l];
    int rc = copy_async(ln.x_slot, x + (size_t)l * Bl * d.latent_elems, (size_t)Bl * d.latent_elems * sizeof(float), st);
    if (rc) return rc;
    fill_i64_kernel<<<(2 * Bl + 127) / 128, 128, 0, st>>>(reinterpret_cast<long long*>(ln.t_slot), 2 * Bl, (long long)t);
    ALDM_CHECK_CUDA(cudaGetLastError());
  }
  if (!d.use_graph) return run_lanes_eager(e, st);
  if (!e->exec) {
    // first use: one eager run (module load, attribute set-up), then capture; the eager run already produced eps
    int rc = run_lanes_eager(e, st);
    if (rc) return rc;
    ALDM_CHECK_CUDA(cudaStreamSynchronize(st));
    return capture_lanes(e);
  }
  ALDM_CHECK_CUDA(cudaGraphLaunch(e->exec, st));
  return ALDM_OK;
}

}  // namespace aldm

using namespace aldm;

extern "C" int aldm_engine_create(const aldm_engine_desc* d, aldm_engine** out) {
  ALDM_REQUIRE(d && out, ALDM_E_ARG, "engine_create: null argument");
  ALDM_REQUIRE(d->n_lanes >= 1 && d->n_lanes <= ALDM_MAX_LANES, ALDM_E_ARG, "engine_create: n_lanes=%d", d->n_lanes);
  ALDM_REQUIRE(d->B > 0 && d->latent_elems > 0 && d->latent_elems % 4 == 0 && d->B % d->n_lanes == 0, ALDM_E_SHAPE,
               "engine_create: B=%d latent_elems=%d n_lanes=%d", d->B, d->latent_elems, d->n_lanes);
  ALDM_REQUIRE(d->n_ctx >= 0 && d->n_ctx <= 2, ALDM_E_SHAPE, "engine_create: n_ctx=%d", d->n_ctx);
  for (int l = 0; l < d->n_lanes; ++l) {
    const aldm_unet_lane& ln = d->lane[l];
    ALDM_REQUIRE(ln.step && ln.x_slot && ln.t_slot && ln.eps_slot, ALDM_E_ARG, "engine_create: lane %d UNet program / slots missing", l);
    for (int i = 0; i < d->n_ctx; ++i)
      ALDM_REQUIRE(ln.ctx_slot[i] && ln.mask_slot[i], ALDM_E_ARG, "engine_create: lane %d context %d slots missing", l, i);
  }
  for (int i = 0; i < d->n_ctx; ++i)
    ALDM_REQUIRE(d->ctx_len[i] > 0 && d->ctx_dim[i] > 0, ALDM_E_ARG, "engine_create: context %d sizes missing", i);
  ALDM_REQUIRE(!d->vae_dec || (d->z_slot && d->mel_slot && d->mel_elems > 0), ALDM_E_ARG, "engine_create: VAE decoder slots missing");
  ALDM_REQUIRE(!d->vocoder || (d->voc_mel_slot && d->wave_slot && d->wave_len > 0 && d->mel_elems > 0), ALDM_E_ARG,
               "engine_create: vocoder slots missing");
  ALDM_REQUIRE(!d->vae_enc || (d->enc_mel_slot && d->moments_slot), ALDM_E_ARG, "engine_create: VAE encoder slots missing");
  aldm_engine* e = new (std::nothrow) aldm_engine();
  ALDM_REQUIRE(e, ALDM_E_NOMEM, "engine_create: out of host memory");
  e->d = *d;
  *out = e;
  return ALDM_OK;
}

extern "C" void aldm_engine_destroy(aldm_engine* e) {
  if (!e) return;
  if (e->exec) cudaGraphExecDestroy(e->exec);
  if (e->graph) cudaGraphDestroy(e->graph);
  if (e->fork) cudaEventDestroy(e->fork);
  for (int l = 0; l < ALDM_MAX_LANES; ++l) {
    if (e->join[l]) cudaEventDestroy(e->join[l]);
    if (e->side[l]) cudaStreamDestroy(e->side[l]);
  }
  delete e;
}

extern "C" int aldm_engine_set_conditioning(aldm_engine* e, int32_t which, const float* ctx0, const float* mask0, int32_t len0,
                                            const float* ctx1, const float* mask1, int32_t len1, const float* film_y,
                                            void* stream) {
  ALDM_REQUIRE(e && (which == 0 || which == 1), ALDM_E_ARG, "set_conditioning: bad engine / half");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const aldm_engine_desc& d = e->d;
  const float* ctx[2] = {ctx0, ctx1};
  const float* msk[2] = {mask0, mask1};
  const int len[2] = {len0, len1};
  const int Bl = d.B / d.n_lanes;
  for (int i = 0; i < d.n_ctx; ++i) {
    ALDM_REQUIRE(ctx[i] && msk[i], ALDM_E_ARG, "set_conditioning: context %d missing", i);
    ALDM_REQUIRE(len[i] >= 1 && len[i] <= d.ctx_len[i], ALDM_E_SHAPE, "set_conditioning: context %d length %d > planned %d", i, len[i],
                 d.ctx_len[i]);
  }
  ALDM_REQUIRE(!d.film_dim || film_y, ALDM_E_ARG, "set_conditioning: film_y missing");
  for (int l = 0; l < d.n_lanes; ++l) {
    const aldm_unet_lane& ln = d.lane[l];
    for (int i = 0; i < d.n_ctx; ++i) {
      float* cdst = ln.ctx_slot[i] + (size_t)which * Bl * d.ctx_len[i] * d.ctx_dim[i];
      float* mdst = ln.mask_slot[i] + (size_t)which * Bl * d.ctx_len[i];
      const float* csrc = ctx[i] + (size_t)l * Bl * len[i] * d.ctx_dim[i];
      const float* msrc = msk[i] + (size_t)l * Bl * len[i];
      // zero-pad to the planned length (padded keys carry mask 0)
      ALDM_CHECK_CUDA(cudaMemsetAsync(cdst, 0, (size_t)Bl * d.ctx_len[i] * d.ctx_dim[i] * sizeof(float), st));
      ALDM_CHECK_CUDA(cudaMemsetAsync(mdst, 0, (size_t)Bl * d.ctx_len[i] * sizeof(float), st));
      ALDM_CHECK_CUDA(cudaMemcpy2DAsync(cdst, (size_t)d.ctx_len[i] * d.ctx_dim[i] * sizeof(float), csrc,
                                        (size_t)len[i] * d.ctx_dim[i] * sizeof(float), (size_t)len[i] * d.ctx_dim[i] * sizeof(float),
                                        Bl, cudaMemcpyDeviceToDevice, st));
      ALDM_CHECK_CUDA(cudaMemcpy2DAsync(mdst, (size_t)d.ctx_len[i] * sizeof(float), msrc, (size_t)len[i] * sizeof(float),
                                        (size_t)len[i] * sizeof(float), Bl, cudaMemcpyDeviceToDevice, st));
    }
    if (d.film_dim) {
      ALDM_REQUIRE(ln.film_slot, ALDM_E_ARG, "set_conditioning: lane %d has no FiLM slot", l);
      int rc = copy_async(ln.film_slot + (size_t)which * Bl * d.film_dim, film_y + (size_t)l * Bl * d.film_dim,
                          (size_t)Bl * d.film_dim * sizeof(float), st);
      if (rc) return rc;
    }
  }
  return ALDM_OK;
}

extern "C" int aldm_engine_precompute(aldm_engine* e, void* stream) {
  ALDM_REQUIRE(e, ALDM_E_ARG, "precompute: null engine");
  for (int l = 0; l < e->d.n_lanes; ++l) {
    if (!e->d.lane[l].cond) continue;
    int rc = aldm_program_run(e->d.lane[l].cond, stream);
    if (rc) return rc;
  }
  return ALDM_OK;
}

extern "C" int aldm_engine_unet_eps(aldm_engine* e, const float* x, int64_t t, float* eps_uncond, float* eps_cond, void* stream) {
  ALDM_REQUIRE(e && x, ALDM_E_ARG, "unet_eps: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = run_unet(e, x, t, st);
  if (rc) return rc;
  const aldm_engine_desc& d = e->d;
  const size_t half = (size_t)(d.B / d.n_lanes) * d.latent_elems;
  for (int l = 0; l < d.n_lanes; ++l) {
    if (eps_uncond && (rc = copy_async(eps_uncond + l * half, d.lane[l].eps_slot, half * sizeof(float), st))) return rc;
    if (eps_cond && (rc = copy_async(eps_cond + l * half, d.lane[l].eps_slot + half, half * sizeof(float), st))) return rc;
  }
  return ALDM_OK;
}

extern "C" int aldm_engine_ddim_step(aldm_engine* e, const float* x, int64_t t, const float* noise, float a_t, float a_prev,
                                     float sigma_t, float sqrt_one_minus_at, float guidance, float* x_prev, float* pred_x0,
                                     void* stream) {
  ALDM_REQUIRE(e && x && noise && x_prev, ALDM_E_ARG, "ddim_step: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = run_unet(e, x, t, st);
  if (rc) return rc;
  const aldm_engine_desc& d = e->d;
  const long long n = (long long)(d.B / d.n_lanes) * d.latent_elems;
  for (int l = 0; l < d.n_lanes; ++l) {
    const float* eps = d.lane[l].eps_slot;
    rc = aldm_ddim_step(x + l * n, eps, eps + n, noise + l * n, x_prev + l * n, pred_x0 ? pred_x0 + l * n : nullptr, n, a_t, a_prev,
                        sigma_t, sqrt_one_minus_at, guidance, stream);
    if (rc) return rc;
  }
  return ALDM_OK;
}

extern "C" int aldm_engine_plms_step(aldm_engine* e, const float* x_in, int64_t t, const float* x_base, const float* held1,
                                     const float* held2, const float* held3, int32_t order, float* e_t_out, float a_t,
                                     float a_prev, float sqrt_one_minus_at, float guidance, float* x_prev, float* pred_x0,
                                     void* stream) {
  ALDM_REQUIRE(e && x_in && x_base && x_prev, ALDM_E_ARG, "plms_step: null argument");
  ALDM_REQUIRE(x_prev != x_base, ALDM_E_ARG, "plms_step: x_prev must not alias x_base");
  // the per-lane kernel checks order and held slots too, but only after the UNet has run: check them before
  ALDM_REQUIRE(order >= ALDM_PLMS_AVERAGE && order <= 4, ALDM_E_ARG, "plms_step: order=%d", order);
  ALDM_REQUIRE(((order != ALDM_PLMS_AVERAGE && order < 2) || held1) && (order < 3 || held2) && (order < 4 || held3),
               ALDM_E_ARG, "plms_step: order %d without the held values it needs", order);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = run_unet(e, x_in, t, st);
  if (rc) return rc;
  const aldm_engine_desc& d = e->d;
  const long long n = (long long)(d.B / d.n_lanes) * d.latent_elems;
  auto at = [&](const float* p, int l) { return p ? p + l * n : nullptr; };
  for (int l = 0; l < d.n_lanes; ++l) {
    const float* eps = d.lane[l].eps_slot;
    rc = aldm_plms_step(x_base + l * n, eps, eps + n, at(held1, l), at(held2, l), at(held3, l), order,
                        e_t_out ? e_t_out + l * n : nullptr, x_prev + l * n, pred_x0 ? pred_x0 + l * n : nullptr, n, a_t,
                        a_prev, sqrt_one_minus_at, guidance, stream);
    if (rc) return rc;
  }
  return ALDM_OK;
}

extern "C" int aldm_engine_vae_decode(aldm_engine* e, const float* z, float* mel, void* stream) {
  ALDM_REQUIRE(e && z && e->d.vae_dec, ALDM_E_ARG, "vae_decode: engine has no decoder program / null z");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = copy_async(e->d.z_slot, z, (size_t)e->d.B * e->d.latent_elems * sizeof(float), st);
  if (rc) return rc;
  if ((rc = aldm_program_run(e->d.vae_dec, stream))) return rc;
  return mel ? copy_async(mel, e->d.mel_slot, (size_t)e->d.B * e->d.mel_elems * sizeof(float), st) : ALDM_OK;
}

extern "C" int aldm_engine_vocoder(aldm_engine* e, const float* mel, float* wave, void* stream) {
  ALDM_REQUIRE(e && mel && e->d.vocoder, ALDM_E_ARG, "vocoder: engine has no vocoder program / null mel");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = copy_async(e->d.voc_mel_slot, mel, (size_t)e->d.B * e->d.mel_elems * sizeof(float), st);
  if (rc) return rc;
  if ((rc = aldm_program_run(e->d.vocoder, stream))) return rc;
  return wave ? copy_async(wave, e->d.wave_slot, (size_t)e->d.B * e->d.wave_len * sizeof(float), st) : ALDM_OK;
}

extern "C" int aldm_engine_vae_encode(aldm_engine* e, const float* mel, float* moments, void* stream) {
  ALDM_REQUIRE(e && mel && e->d.vae_enc, ALDM_E_ARG, "vae_encode: engine has no encoder program / null mel");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = copy_async(e->d.enc_mel_slot, mel, (size_t)e->d.B * e->d.mel_elems * sizeof(float), st);
  if (rc) return rc;
  if ((rc = aldm_program_run(e->d.vae_enc, stream))) return rc;
  return moments ? copy_async(moments, e->d.moments_slot, (size_t)e->d.B * 2 * e->d.latent_elems * sizeof(float), st) : ALDM_OK;
}

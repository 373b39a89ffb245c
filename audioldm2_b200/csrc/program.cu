// Program executor: a flat table of aldm_op records (built by the Python planner from the
// reference config + state_dict) replayed on a stream, or captured once into a CUDA graph and
// re-launched per DDIM step (~900 kernels per UNet evaluation; the reference issues ~3,700 per step
// from Python).  Also the misc C-ABI entry points (error string, ABI self-description).
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "common.cuh"

namespace aldm {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;      // H100 SXM
  }
  return n;
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("ALDM_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

int gemm_launch(const aldm_gemm_desc& d, cudaStream_t st);
int gemm_num_launches(const aldm_gemm_desc& d);
int prep_launch(const aldm_prep_desc& d, cudaStream_t st);
int prep_num_launches(const aldm_prep_desc& d);
int attention_launch(const aldm_attn_desc& d, cudaStream_t st);
int kv_attention_launch(const aldm_kv_attn_desc& d, cudaStream_t st);
int seq_assemble_launch(const aldm_seq_assemble_desc& d, cudaStream_t st);
int seq_feedback_launch(const aldm_seq_feedback_desc& d, cudaStream_t st);
int t5_embed_launch(const aldm_t5_embed_desc& d, cudaStream_t st);
int t5_rmsnorm_launch(const aldm_t5_rmsnorm_desc& d, cudaStream_t st);
int t5_attention_launch(const aldm_t5_attn_desc& d, cudaStream_t st);
int t5_gate_launch(const aldm_t5_gate_desc& d, cudaStream_t st);
int clap_embed_launch(const aldm_clap_embed_desc& d, cudaStream_t st);
int clap_layernorm_launch(const aldm_clap_ln_desc& d, cudaStream_t st);
int clap_attention_launch(const aldm_clap_attn_desc& d, cudaStream_t st);
int clap_gelu_launch(const aldm_clap_gelu_desc& d, cudaStream_t st);
int clap_head_launch(const aldm_clap_head_desc& d, cudaStream_t st);
int htsat_logmel_launch(const aldm_htsat_logmel_desc& d, cudaStream_t st);
int htsat_patch_launch(const aldm_htsat_patch_desc& d, cudaStream_t st);
int htsat_window_attention_launch(const aldm_htsat_attn_desc& d, cudaStream_t st);
int htsat_merge_launch(const aldm_htsat_merge_desc& d, cudaStream_t st);
int htsat_head_launch(const aldm_htsat_head_desc& d, cudaStream_t st);

}  // namespace aldm

struct aldm_program {
  std::vector<aldm_op> ops;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
};

using namespace aldm;

static int run_op(const aldm_op& op, cudaStream_t st) {
  switch (op.kind) {
    case ALDM_OP_GEMM: return gemm_launch(op.u.gemm, st);
    case ALDM_OP_PREP: return prep_launch(op.u.prep, st);
    case ALDM_OP_ATTN: return attention_launch(op.u.attn, st);
    case ALDM_OP_SOFTMAX:
      return aldm_softmax_rows(op.u.softmax.x, op.u.softmax.rows, op.u.softmax.n, op.u.softmax.scale, op.u.softmax.out_hi,
                               op.u.softmax.out_lo, st);
    case ALDM_OP_TEMB:
      return aldm_timestep_embedding(op.u.temb.t, op.u.temb.B, op.u.temb.dim, op.u.temb.freqs, op.u.temb.out_hi,
                                     op.u.temb.out_lo, st);
    case ALDM_OP_TRANSPOSE:
      return aldm_transpose_chw(op.u.transpose.src, op.u.transpose.dst, op.u.transpose.B, op.u.transpose.C,
                                op.u.transpose.HW, op.u.transpose.to_nhwc, st);
    case ALDM_OP_PACKB:
      return aldm_pack_b(op.u.packb.src, op.u.packb.lds, op.u.packb.transpose, op.u.packb.N, op.u.packb.K, op.u.packb.bn,
                         op.u.packb.dst_packed, op.u.packb.dst_plain, st);
    case ALDM_OP_SEQ_ASSEMBLE: return seq_assemble_launch(op.u.seq_assemble, st);
    case ALDM_OP_KV_ATTN: return kv_attention_launch(op.u.kv_attn, st);
    case ALDM_OP_SEQ_FEEDBACK: return seq_feedback_launch(op.u.seq_feedback, st);
    case ALDM_OP_T5_EMBED: return t5_embed_launch(op.u.t5_embed, st);
    case ALDM_OP_T5_RMSNORM: return t5_rmsnorm_launch(op.u.t5_rmsnorm, st);
    case ALDM_OP_T5_ATTN: return t5_attention_launch(op.u.t5_attn, st);
    case ALDM_OP_T5_GATE: return t5_gate_launch(op.u.t5_gate, st);
    case ALDM_OP_CLAP_EMBED: return clap_embed_launch(op.u.clap_embed, st);
    case ALDM_OP_CLAP_LN: return clap_layernorm_launch(op.u.clap_ln, st);
    case ALDM_OP_CLAP_ATTN: return clap_attention_launch(op.u.clap_attn, st);
    case ALDM_OP_CLAP_GELU: return clap_gelu_launch(op.u.clap_gelu, st);
    case ALDM_OP_CLAP_HEAD: return clap_head_launch(op.u.clap_head, st);
    case ALDM_OP_HTSAT_LOGMEL: return htsat_logmel_launch(op.u.htsat_logmel, st);
    case ALDM_OP_HTSAT_PATCH: return htsat_patch_launch(op.u.htsat_patch, st);
    case ALDM_OP_HTSAT_ATTN: return htsat_window_attention_launch(op.u.htsat_attn, st);
    case ALDM_OP_HTSAT_MERGE: return htsat_merge_launch(op.u.htsat_merge, st);
    case ALDM_OP_HTSAT_HEAD: return htsat_head_launch(op.u.htsat_head, st);
    case ALDM_OP_COPY:
      ALDM_CHECK_CUDA(cudaMemcpyAsync(op.u.copy.dst, op.u.copy.src, (size_t)op.u.copy.bytes, cudaMemcpyDeviceToDevice, st));
      return ALDM_OK;
    default:
      set_error("program: unknown op kind %d", op.kind);
      return ALDM_E_ARG;
  }
}

extern "C" int aldm_program_create(const aldm_op* ops, int32_t n_ops, aldm_program** out) {
  ALDM_REQUIRE(ops && out && n_ops > 0, ALDM_E_ARG, "program_create: bad arguments");
  aldm_program* p = new (std::nothrow) aldm_program();
  ALDM_REQUIRE(p, ALDM_E_NOMEM, "program_create: out of host memory");
  p->ops.assign(ops, ops + n_ops);
  *out = p;
  return ALDM_OK;
}

extern "C" int aldm_program_run_range(aldm_program* p, int32_t first, int32_t last, void* stream) {
  ALDM_REQUIRE(p, ALDM_E_ARG, "program_run: null program");
  ALDM_REQUIRE(first >= 0 && last <= (int)p->ops.size() && first <= last, ALDM_E_ARG, "program_run: bad range %d..%d", first, last);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int i = first; i < last; ++i) {
    int rc = run_op(p->ops[i], st);
    if (rc != ALDM_OK) {
      char tmp[900];
      strncpy(tmp, g_err, sizeof(tmp) - 1);
      tmp[sizeof(tmp) - 1] = 0;
      set_error("op %d (kind %d, tag %d): %s", i, p->ops[i].kind, p->ops[i].tag, tmp);
      return rc;
    }
  }
  return ALDM_OK;
}

extern "C" int aldm_program_run(aldm_program* p, void* stream) {
  ALDM_REQUIRE(p, ALDM_E_ARG, "program_run: null program");
  return aldm_program_run_range(p, 0, (int32_t)p->ops.size(), stream);
}

extern "C" int aldm_program_capture(aldm_program* p, void* stream) {
  ALDM_REQUIRE(p, ALDM_E_ARG, "program_capture: null program");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (p->exec) { cudaGraphExecDestroy(p->exec); p->exec = nullptr; }
  if (p->graph) { cudaGraphDestroy(p->graph); p->graph = nullptr; }
  ALDM_CHECK_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  int rc = aldm_program_run(p, stream);
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamEndCapture(st, &g);
  if (rc != ALDM_OK) { if (g) cudaGraphDestroy(g); return rc; }
  if (e != cudaSuccess) { set_error("program_capture: end capture: %s", cudaGetErrorString(e)); return ALDM_E_CUDA; }
  p->graph = g;
  ALDM_CHECK_CUDA(cudaGraphInstantiate(&p->exec, p->graph, 0));
  return ALDM_OK;
}

extern "C" int aldm_program_replay(aldm_program* p, void* stream) {
  ALDM_REQUIRE(p && p->exec, ALDM_E_ARG, "program_replay: program not captured");
  ALDM_CHECK_CUDA(cudaGraphLaunch(p->exec, reinterpret_cast<cudaStream_t>(stream)));
  return ALDM_OK;
}

extern "C" int aldm_program_is_captured(aldm_program* p) { return (p && p->exec) ? 1 : 0; }

extern "C" int aldm_program_num_launches(aldm_program* p) {
  if (!p) return 0;
  int n = 0;
  for (const aldm_op& op : p->ops) {
    if (op.kind == ALDM_OP_GEMM) n += gemm_num_launches(op.u.gemm);
    else if (op.kind == ALDM_OP_PREP) n += prep_num_launches(op.u.prep);
    else if (op.kind == ALDM_OP_COPY) n += 0;
    else n += 1;
  }
  return n;
}

extern "C" void aldm_program_destroy(aldm_program* p) {
  if (!p) return;
  if (p->exec) cudaGraphExecDestroy(p->exec);
  if (p->graph) cudaGraphDestroy(p->graph);
  delete p;
}

extern "C" int aldm_abi_version(void) { return ALDM_ABI_VERSION; }
extern "C" size_t aldm_sizeof_op(void) { return sizeof(aldm_op); }
extern "C" size_t aldm_sizeof_gemm_desc(void) { return sizeof(aldm_gemm_desc); }
extern "C" size_t aldm_offsetof_gemm(int32_t field) {
  switch (field) {
    case 0: return offsetof(aldm_gemm_desc, B);
    case 1: return offsetof(aldm_gemm_desc, ntaps);
    case 2: return offsetof(aldm_gemm_desc, dy);
    case 3: return offsetof(aldm_gemm_desc, N);
    case 4: return offsetof(aldm_gemm_desc, ldo);
    case 5: return offsetof(aldm_gemm_desc, act);
    case 6: return offsetof(aldm_gemm_desc, alpha);
    case 7: return offsetof(aldm_gemm_desc, n_split);
    default: return (size_t)-1;
  }
}
extern "C" size_t aldm_sizeof_engine_desc(void) { return sizeof(aldm_engine_desc); }
extern "C" const char* aldm_last_error(void) { return g_err; }

extern "C" int aldm_device_check(int32_t device) {
  cudaDeviceProp prop;
  ALDM_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  ALDM_REQUIRE(prop.major == 9 && prop.minor == 0, ALDM_E_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device,
               prop.major, prop.minor);
  return ALDM_OK;
}

// capi.cu -- C-ABI plumbing shared by every entry point: thread-local error text, launch counter,
// device query, and the stand-alone RoPE entry (which owns a small cache of cos/sin tables).
#include <stdarg.h>
#include <ctype.h>
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "ops.h"

namespace sb {

static thread_local char g_err[1024] = "";
static thread_local int64_t g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches += n; }
int set_option(const char* key, int value);

struct ProfRec { cudaEvent_t a, b; int kind; double flops; };
static thread_local bool g_prof_on = false;
static thread_local std::vector<ProfRec>* g_prof = nullptr;

bool profile_enabled() { return g_prof_on; }
void profile_mark_begin(int kind, cudaStream_t stream) {
  if (!g_prof_on) return;
  ProfRec r;
  r.kind = kind; r.flops = 0.0;
  cudaEventCreate(&r.a); cudaEventCreate(&r.b);
  cudaEventRecord(r.a, stream);
  g_prof->push_back(r);
}
void profile_mark_end(int kind, cudaStream_t stream, double flops) {
  if (!g_prof_on || g_prof->empty()) return;
  ProfRec& r = g_prof->back();
  r.flops = flops;
  cudaEventRecord(r.b, stream);
}

static std::map<std::string, int>& options() {
  static std::map<std::string, int> o = [] {
    std::map<std::string, int> m = {{"decode_pdl", 1}, {"gemv_ksplit", 0},
                                    {"encoder_ln_fold", 1}, {"gemv_prefetch_mb", 0}, {"encoder_stats_fused", 1}, {"gemm_sched", 1}, {"decode_fused_attention", 1}, {"gemv_no_allocate", 1}};
    // A/B runs of unmodified commands (bench.py): SEEDB200_OPT_<KEY>=<int> overrides a default at load time
    for (auto& kv : m) {
      std::string env = "SEEDB200_OPT_";
      for (char ch : kv.first) env += (char)toupper((unsigned char)ch);
      if (const char* v = getenv(env.c_str())) kv.second = atoi(v);
    }
    return m;
  }();
  return o;
}
static long long g_dbg_ptr = 0;
long long get_option64(const char* key) { return std::string(key) == "vit_attention_dbg_ptr" ? g_dbg_ptr : 0; }
int get_option(const char* key) {
  auto it = options().find(key);
  return it == options().end() ? 0 : it->second;
}
int set_option(const char* key, int value) {
  auto it = options().find(key);
  if (it == options().end()) {
    set_error("unknown option '%s'", key);
    return SEEDB200_ERR_INVALID;
  }
  it->second = value;
  return 0;
}

static thread_local bool g_pdl_scope = false;
bool pdl_scope_active() { return g_pdl_scope; }
void pdl_scope_set(bool on) { g_pdl_scope = on; }

int cur_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= SB_MAX_DEVICES) dev = 0;
  return dev;
}

int num_sms() {
  static int sms_dev[SB_MAX_DEVICES] = {};
  const int dev = cur_device();
  int& sms = sms_dev[dev];
  if (sms == 0) {
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 148;
  }
  return sms;
}

struct RopeTables { void* cos_t; void* sin_t; int max_pos; };
static std::mutex g_rope_mu;
static std::map<long long, RopeTables> g_rope_cache;

int get_rope_tables(int D, float base, int min_pos, const void** cos_t, const void** sin_t, int* max_pos,
                    cudaStream_t stream) {
  std::lock_guard<std::mutex> lk(g_rope_mu);
  int dev = 0;
  SB_CHECK_CUDA(cudaGetDevice(&dev));
  const long long key = ((long long)dev << 48) | ((long long)D << 32) | (long long)(unsigned)(base);
  auto it = g_rope_cache.find(key);
  if (it != g_rope_cache.end() && it->second.max_pos >= min_pos) {
    *cos_t = it->second.cos_t; *sin_t = it->second.sin_t; *max_pos = it->second.max_pos;
    return 0;
  }
  int n = 4096;
  while (n < min_pos) n *= 2;
  RopeTables t;
  t.max_pos = n;
  SB_CHECK_CUDA(cudaMalloc(&t.cos_t, (size_t)n * (D / 2) * 2));
  SB_CHECK_CUDA(cudaMalloc(&t.sin_t, (size_t)n * (D / 2) * 2));
  SB_PROPAGATE(build_rope_tables(t.cos_t, t.sin_t, n, D, base, stream));
  // later callers may use the table from other streams: publish it only once the build has finished
  SB_CHECK_CUDA(cudaStreamSynchronize(stream));
  g_rope_cache[key] = t;   // an older, smaller table (if any) stays alive: in-flight kernels may still read it
  *cos_t = t.cos_t; *sin_t = t.sin_t; *max_pos = n;
  return 0;
}

}  // namespace sb

extern "C" {

int seedb200_version(void) { return SEEDB200_VERSION; }
const char* seedb200_last_error(void) { return sb::g_err; }
int64_t seedb200_launch_count(void) { return sb::g_launches; }
void seedb200_reset_launch_count(void) { sb::g_launches = 0; }

int seedb200_set_option(const char* key, int value) {
  if (key == nullptr) {
    sb::set_error("set_option: null key");
    return SEEDB200_ERR_INVALID;
  }
  return sb::set_option(key, value);
}

/* debug only (not declared in seedb200.h): device buffer that receives the attention kernel's timeline */
void seedb200_debug_set_attn_timeline(void* dev_ptr) { sb::g_dbg_ptr = (long long)(uintptr_t)dev_ptr; }

static int seedb200_set_option_unused(const char* key, int value) {
  return sb::set_option(key, value);
}

int seedb200_profile_begin(void) {
  if (sb::g_prof == nullptr) sb::g_prof = new std::vector<sb::ProfRec>();
  sb::g_prof->clear();
  sb::g_prof_on = true;
  return 0;
}
int seedb200_profile_end(double* out6) {
  if (!sb::g_prof_on || out6 == nullptr) {
    sb::set_error("profile_end without profile_begin");
    return SEEDB200_ERR_INVALID;
  }
  sb::g_prof_on = false;
  SB_CHECK_CUDA(cudaDeviceSynchronize());
  for (int i = 0; i < 6; ++i) out6[i] = 0.0;
  for (auto& r : *sb::g_prof) {
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, r.a, r.b);
    if (r.kind >= 0 && r.kind < 2) {
      out6[r.kind * 3 + 0] += 1.0;
      out6[r.kind * 3 + 1] += ms;
      out6[r.kind * 3 + 2] += r.flops;
    }
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  sb::g_prof->clear();
  return 0;
}

int seedb200_rope_kv_append(const void* qkv, const int64_t* positions, int B, int S, int H, int D, int past_len,
                            int max_seq, void* q_out, void* k_cache, void* v_cache, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const void *cos_t, *sin_t;
  int max_pos;
  SB_PROPAGATE(sb::get_rope_tables(D, 10000.0f, max_seq, &cos_t, &sin_t, &max_pos, st));
  return sb::rope_kv_append_tables(qkv, positions, B, S, H, D, past_len, max_seq, max_pos, cos_t, sin_t, q_out,
                                   k_cache, v_cache, st);
}

/* the fused decode form: RoPE + append + attention of one new token per sequence, one launch */
int seedb200_decode_attention_rope(const void* qkv, const int64_t* positions, int B, int H, int D, int past_len,
                                   int max_seq, void* k_cache, void* v_cache, void* out, float scale, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const void *cos_t, *sin_t;
  int max_pos;
  SB_PROPAGATE(sb::get_rope_tables(D, 10000.0f, max_seq, &cos_t, &sin_t, &max_pos, st));
  return sb::decode_attention_rope(qkv, positions, B, H, D, past_len, max_seq, max_pos, cos_t, sin_t, k_cache, v_cache,
                                   out, scale, st);
}

int seedb200_decode_attention_rope_lineage(const void* qkv, const int64_t* positions, const int32_t* slot, int B, int H,
                                           int D, int past_len, int max_seq, void* k_cache, void* v_cache, void* out,
                                           float scale, void* stream) {
  SB_REQUIRE(slot != nullptr, "seedb200_decode_attention_rope_lineage: null slot table");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const void *cos_t, *sin_t;
  int max_pos;
  SB_PROPAGATE(sb::get_rope_tables(D, 10000.0f, max_seq, &cos_t, &sin_t, &max_pos, st));
  return sb::decode_attention_rope(qkv, positions, B, H, D, past_len, max_seq, max_pos, cos_t, sin_t, k_cache, v_cache,
                                   out, scale, st, nullptr, slot);
}

}  // extern "C"

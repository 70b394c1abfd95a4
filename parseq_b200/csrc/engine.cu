// libparseq_b200.so: host-side engine + C ABI (include/parseq_b200.h) of the H100-native (sm_90a) PARSeq
// inference path.  Restates, as a fixed kernel schedule on one CUDA stream, what
// strhub/models/parseq/model.py:105-169 (PARSeq.forward: encode, AR loop, NAR, cloze refinement)
// does through nn.Module calls.  There is no CPU path: without an sm_90 device creation fails.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/parseq_b200.h"
#include "gemm.cuh"
#include "kernels.cuh"
#include "dec_ar.cuh"
#include "dec_ar2.cuh"
#include "gemm_ln.cuh"
#include "mlp_ln.cuh"
#include "attn_wgmma.cuh"
#include "qkv_attn.cuh"
#include "crops.cuh"
#include "regions.cuh"
#include "orient.cuh"
#include "owners.h"

namespace {

constexpr int kMaxHeadClasses = 16384;    // num_tokens - 2 (parseq_create)
constexpr int kMaxLabelLength = 63;       // L = max_label_length + 1 <= 64 decode positions (parseq_create)

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
#define PQ_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return fail(PARSEQ_ERR_CUDA, std::string(#expr) + " -> " + cudaGetErrorString(_e));          \
  } while (0)
#define PQ_TRY(expr)                 \
  do {                               \
    int _r = (expr);                 \
    if (_r != PARSEQ_OK) return _r;  \
  } while (0)

// ---------------------------------------------------------------- driver entry point for TMA descriptors
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled g_encode = nullptr;

int load_driver_api() {
  if (g_encode != nullptr) return PARSEQ_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess)
    return fail(PARSEQ_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  return PARSEQ_OK;
}

// 2D tensor map: rows x cols (cols contiguous), row stride ld elements, box = box_rows x box_cols (box_cols * esize
// = 128 B), 128B swizzle.  esize 2 = bf16, 4 = fp32.
int make_tmap(CUtensorMap* tm, const void* ptr, int esize, long long rows, long long cols, long long ld, int box_cols,
              int box_rows) {
  PQ_TRY(load_driver_api());
  if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0 || ((ld * esize) & 15) != 0)
    return fail(PARSEQ_ERR_INVALID_ARG, "GEMM operand must be 16-byte aligned with a 16-byte multiple row stride");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * static_cast<cuuint64_t>(esize)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(tm, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                        const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(PARSEQ_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string(int(r)));
  return PARSEQ_OK;
}

// 3D bf16 tensor map [d2][d1][d0] (d0 contiguous), strides in elements, box = box_d0 x box_d1 x 1, 128B swizzle.
// Rows past d1 read as zeros.
int make_tmap3d(CUtensorMap* tm, const void* ptr, long long d0, long long d1, long long d2, long long ld1, long long ld2,
                int box_d0, int box_d1) {
  PQ_TRY(load_driver_api());
  if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0 || ((ld1 * 2) & 15) != 0 || ((ld2 * 2) & 15) != 0)
    return fail(PARSEQ_ERR_INVALID_ARG, "tensor map operand must be 16-byte aligned with 16-byte multiple strides");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1), static_cast<cuuint64_t>(d2)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld1) * 2u, static_cast<cuuint64_t>(ld2) * 2u};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box_d0), static_cast<cuuint32_t>(box_d1), 1u};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(PARSEQ_ERR_CUDA, "cuTensorMapEncodeTiled(3d) failed: " + std::to_string(int(r)));
  return PARSEQ_OK;
}

// The decoder's column-blocked cross K/V cache [2D/64][kv_rows = max_batch * T][64] bf16 viewed as the 4D tensor
// [2D/64][max_batch][T][64]: a box of {64, box_t, 1, 1} at (0, key0, image, panel) holds keys key0.. of ONE image, and
// the keys past T of that image read as zeros (never the next image's keys, nor rows past the cache), so the softmax's
// P = 0 for a masked key never meets a non-finite V.  128B swizzle.
int make_tmap_kv4d(CUtensorMap* tm, const void* ptr, int T, int max_batch, int panels, int box_t) {
  PQ_TRY(load_driver_api());
  if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0)
    return fail(PARSEQ_ERR_INVALID_ARG, "tensor map operand must be 16-byte aligned");
  const cuuint64_t row = 128;                               // 64 bf16
  cuuint64_t dims[4] = {64, static_cast<cuuint64_t>(T), static_cast<cuuint64_t>(max_batch), static_cast<cuuint64_t>(panels)};
  cuuint64_t strides[3] = {row, row * T, row * T * max_batch};
  cuuint32_t box[4] = {64, static_cast<cuuint32_t>(box_t), 1u, 1u};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = g_encode(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(PARSEQ_ERR_CUDA, "cuTensorMapEncodeTiled(K/V 4d) failed: " + std::to_string(int(r)));
  return PARSEQ_OK;
}

uint16_t f32_to_bf16_rne(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40u);  // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return static_cast<uint16_t>(u >> 16);
}

// Launch options.  Every engine handle owns one (parseq_set_option(handle, ...)); `g_default_opts` serves only the
// bare kernel exports (parseq_gemm_bf16 & co., unit tests) and parseq_set_option(NULL, ...).
struct LaunchOpts {
  int sm_count = 0;
  bool use_pdl = true;          // programmatic dependent launch on every kernel of the forward chain
  int ln_cta_group = 0;         // fused GEMM + LayerNorm full-row kernel: 2 = CTA pairs (MODE 1), else single CTAs (MODE 0)
  int ln_split = 0;             // fused GEMM + LayerNorm: 2 = persistent column-split CTA pairs (gemm_ln.cuh MODE 2), 0 = auto (MODE 2 at D = 384), 1 = never
  int mlp_cta_group = 0;        // one-kernel MLP (mlp_ln.cuh): 0 = auto (pairs), 1 / 2 = forced
  bool pair_pdl = false;        // experiments: programmatic dependent launch also on CTA-pair (cluster) launches
  int gemm_stages = 0;          // experiments: cap the operand ring depth (0 = full)
  int attn_impl = 0;            // 0: mma.sync kernels (kernels.cuh), the faster on H100; 1: wgmma kernel (attn_wgmma.cuh)
  int ln_clusters = 0;          // co-resident clusters of the persistent GEMM + LayerNorm kernel (0: not queried yet)
};
LaunchOpts g_default_opts;

int ensure_sm_count(LaunchOpts& o) {
  if (o.sm_count == 0) {
    int dev = 0;
    PQ_CUDA(cudaGetDevice(&dev));
    PQ_CUDA(cudaDeviceGetAttribute(&o.sm_count, cudaDevAttrMultiProcessorCount, dev));
  }
  return PARSEQ_OK;
}

// The configuration of one cudaLaunchKernelEx call.  cluster > 0 sets a cluster dimension of cluster x 1 x 1 (a cluster
// of 1 is an explicit attribute too); pdl allows programmatic dependent launch (the kernels call
// griddepcontrol.{launch_dependents,wait}).  Not copyable: `cfg.attrs` points into the object.  The occupancy queries
// take `cfg` as well.
struct LaunchConfig {
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[2];
  LaunchConfig(dim3 grid, dim3 block, size_t smem, cudaStream_t st, unsigned cluster, bool pdl) {
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr;
    if (cluster > 0) {
      attr[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
      attr[cfg.numAttrs].val.clusterDim.x = cluster;
      attr[cfg.numAttrs].val.clusterDim.y = 1;
      attr[cfg.numAttrs].val.clusterDim.z = 1;
      ++cfg.numAttrs;
    }
    if (pdl) {
      attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
      ++cfg.numAttrs;
    }
  }
  LaunchConfig(const LaunchConfig&) = delete;
  LaunchConfig& operator=(const LaunchConfig&) = delete;
};

template <typename... KArgs, typename... Args>
int launch_ex(const LaunchConfig& lc, void (*kern)(KArgs...), const Args&... args) {
  PQ_CUDA(cudaLaunchKernelEx(&lc.cfg, kern, static_cast<KArgs>(args)...));
  return PARSEQ_OK;
}
// a launch without a cluster attribute, with PDL as the options say
template <typename... KArgs, typename... Args>
int launch_k(const LaunchOpts& lo, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Args&... args) {
  return launch_ex(LaunchConfig(grid, block, smem, st, 0, lo.use_pdl), kern, args...);
}
// PDL on a launch of cg-CTA clusters of the forward chain: CTA pairs take it only with the "pair_pdl" option
bool cluster_pdl(const LaunchOpts& lo, int cg) { return lo.use_pdl && (cg == 1 || lo.pair_pdl); }

// Calls f(std::integral_constant<int, D>) for the embedding widths the kernels are instantiated for.
template <typename F>
int dispatch_width(int D, const char* what, F&& f) {
  switch (D) {
    case 192: return f(std::integral_constant<int, 192>{});
    case 384: return f(std::integral_constant<int, 384>{});
    case 768: return f(std::integral_constant<int, 768>{});
    default: return fail(PARSEQ_ERR_UNSUPPORTED, std::string(what) + ": embed_dim must be 192, 384 or 768");
  }
}

template <int EPI, int STORE>
int launch_gemm_cfg(const LaunchOpts& lo, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to,
                    const pq::GemmParams& p, int tiles, cudaStream_t st) {
  const int grid = tiles < lo.sm_count ? tiles : lo.sm_count;   // persistent: one CTA per SM, tiles strided
  return launch_k(lo, pq::gemm_bf16_wgmma_kernel<EPI, STORE>, dim3(static_cast<unsigned>(grid)), dim3(pq::GEMM_THREADS),
                  pq::GemmCfg::smem_bytes<STORE != pq::ST_REG>(), st, ta, tb, to, p);
}

size_t head_smem_bytes(int C, int D) {
  return ((static_cast<size_t>(C) * (D / 2 + 1) * 4 + 15) / 16) * 16 + static_cast<size_t>(pq::HEAD_ROWS) * D * 4 +
         4 * pq::HEAD_ROWS * 128 * 4 + pq::HEAD_ROWS * 128 * 4;
}
int ln_head_argmax_launch(const LaunchOpts& lo, const float* y, const float* g, const float* b, float eps, const __nv_bfloat16* Wh, const float* bh,
                          int M, int C, int D, float* logits, long long logits_ld, int* ids, int ids_ld, int nq, int dst_off,
                          const int* forced, int forced_ld, const uint32_t* mask, cudaStream_t st) {
  if (C > 128) return fail(PARSEQ_ERR_UNSUPPORTED, "head kernel covers at most 128 classes");
  const dim3 grid((M + pq::HEAD_ROWS - 1) / pq::HEAD_ROWS), block(384);
  const size_t sm = head_smem_bytes(C, D);
  switch (D) {
    case 192: return launch_k(lo, pq::dec_ln_head_argmax_kernel<192>, grid, block, sm, st, y, g, b, eps, Wh, bh, M, C, logits,
                              logits_ld, ids, ids_ld, nq, dst_off, forced, forced_ld, mask);
    case 384: return launch_k(lo, pq::dec_ln_head_argmax_kernel<384>, grid, block, sm, st, y, g, b, eps, Wh, bh, M, C, logits,
                              logits_ld, ids, ids_ld, nq, dst_off, forced, forced_ld, mask);
    case 768: return launch_k(lo, pq::dec_ln_head_argmax_kernel<768>, grid, block, sm, st, y, g, b, eps, Wh, bh, M, C, logits,
                              logits_ld, ids, ids_ld, nq, dst_off, forced, forced_ld, mask);
    default: return fail(PARSEQ_ERR_UNSUPPORTED, "head kernel: embed_dim must be 192, 384 or 768");
  }
}

// the cluster AR kernel of a head width and id row pitch: WIDE (> 128 classes) is the class-sliced head; IDP = 64 holds
// labels of up to 63 characters (L <= 64), IDP = 32 the rest
template <int D, int MT, int CS, bool HS, bool WIDE, int IDP>
constexpr auto ar2_kernel() {
  if constexpr (IDP == 64) {
    if constexpr (WIDE) return pq::dec_ar2_long_wide_kernel<D, MT, CS, HS>;
    else return pq::dec_ar2_long_kernel<D, MT, CS, HS>;
  } else {
    if constexpr (WIDE) return pq::dec_ar2_wide_kernel<D, MT, CS, HS>;
    else return pq::dec_ar2_kernel<D, MT, CS, HS>;
  }
}
template <typename... KArgs>
int set_smem(void (*kern)(KArgs...), size_t bytes) {
  PQ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
  return PARSEQ_OK;
}
template <int D, int MT, int CS, bool WIDE, int IDP>
int ar2_attr() {
  PQ_TRY(set_smem(ar2_kernel<D, MT, CS, false, WIDE, IDP>(), pq::dec_ar2_smem_bytes<D, MT, CS, IDP>()));
  if constexpr (MT == 1 && CS == 8 && D / 64 <= CS)      // head-split variant for tiny batches
    PQ_TRY(set_smem(ar2_kernel<D, MT, CS, true, WIDE, IDP>(), pq::dec_ar2_smem_bytes<D, MT, CS, IDP>()));
  return PARSEQ_OK;
}
template <bool WIDE, int IDP>
int ar2_set_attributes() {
  PQ_TRY((ar2_attr<192, 1, 8, WIDE, IDP>())); PQ_TRY((ar2_attr<192, 2, 8, WIDE, IDP>())); PQ_TRY((ar2_attr<384, 1, 8, WIDE, IDP>()));
  PQ_TRY((ar2_attr<384, 2, 8, WIDE, IDP>())); PQ_TRY((ar2_attr<768, 1, 8, WIDE, IDP>()));
  PQ_TRY((ar2_attr<192, 1, 6, WIDE, IDP>())); PQ_TRY((ar2_attr<192, 2, 6, WIDE, IDP>())); PQ_TRY((ar2_attr<384, 1, 6, WIDE, IDP>()));
  PQ_TRY((ar2_attr<384, 2, 6, WIDE, IDP>())); PQ_TRY((ar2_attr<768, 1, 6, WIDE, IDP>()));
  return PARSEQ_OK;
}

template <int D, int MODE>
int gemm_ln_attr() { return set_smem(pq::gemm_ln_fused_kernel<D, MODE>, pq::GemmLnCfg<D, MODE>::kSmemBytes); }
template <int D, int CG>
int mlp_ln_attr() { return set_smem(pq::mlp_ln_fused_kernel<D, CG>, pq::MlpLnCfg<D, CG>::kSmemBytes); }
template <int NK>
int attn_wgmma_attr() { return set_smem(pq::enc_attention_wgmma_kernel<NK>, pq::atw_smem_bytes<NK>()); }
template <int D>
int qkv_attn_attr() { return set_smem(pq::enc_qkv_attn_kernel<D>, pq::QkvAttnCfg::kSmemBytes); }
template <int EPI, int STORE>
int gemm_attr() { return set_smem(pq::gemm_bf16_wgmma_kernel<EPI, STORE>, pq::GemmCfg::smem_bytes<STORE != pq::ST_REG>()); }
constexpr int kTmaBenchSmem = 12 * pq::A2_SLOT + 1024 + 256;

// The dynamic shared memory limit of every engine kernel that needs more than the default.  cudaFuncSetAttribute acts on
// the current device and must not run under stream capture: call through ensure_kernel_attributes.
int init_kernel_attributes() {
  PQ_TRY(set_smem(pq::dec_ar_kernel<192, 1>, pq::dec_ar_smem_bytes<192>()));
  PQ_TRY(set_smem(pq::dec_ar_kernel<192, 2>, pq::dec_ar_smem_bytes<192>()));
  PQ_TRY(set_smem(pq::dec_ar_kernel<384, 1>, pq::dec_ar_smem_bytes<384>()));
  PQ_TRY(set_smem(pq::dec_ar_kernel<384, 2>, pq::dec_ar_smem_bytes<384>()));
  PQ_TRY(set_smem(pq::dec_ar_kernel<768, 1>, pq::dec_ar_smem_bytes<768>()));
  PQ_TRY(set_smem(pq::dec_ar_kernel<768, 2>, pq::dec_ar_smem_bytes<768>()));
  PQ_TRY((ar2_set_attributes<false, 32>()));
  PQ_TRY((ar2_set_attributes<true, 32>()));
  PQ_TRY((ar2_set_attributes<false, 64>()));
  PQ_TRY((ar2_set_attributes<true, 64>()));
  PQ_TRY(set_smem(pq::dec_ln_head_argmax_kernel<192>, 120 * 1024));
  PQ_TRY(set_smem(pq::dec_ln_head_argmax_kernel<384>, 160 * 1024));
  PQ_TRY(set_smem(pq::dec_ln_head_argmax_kernel<768>, 226 * 1024));
  PQ_TRY((gemm_ln_attr<192, 0>())); PQ_TRY((gemm_ln_attr<384, 0>())); PQ_TRY((gemm_ln_attr<192, 1>()));
  PQ_TRY((gemm_ln_attr<384, 1>())); PQ_TRY((gemm_ln_attr<384, 2>()));
  PQ_TRY((mlp_ln_attr<192, 1>())); PQ_TRY((mlp_ln_attr<384, 1>())); PQ_TRY((mlp_ln_attr<192, 2>())); PQ_TRY((mlp_ln_attr<384, 2>()));
  PQ_TRY((attn_wgmma_attr<128>())); PQ_TRY((attn_wgmma_attr<256>()));
  PQ_TRY((qkv_attn_attr<192>())); PQ_TRY((qkv_attn_attr<384>()));
  PQ_TRY((gemm_attr<pq::EPI_F32, pq::ST_REG>()));
  PQ_TRY((gemm_attr<pq::EPI_F32_RESID, pq::ST_REG>()));
  PQ_TRY((gemm_attr<pq::EPI_BF16, pq::ST_REG>()));
  PQ_TRY((gemm_attr<pq::EPI_BF16, pq::ST_TMA_2D>()));
  PQ_TRY((gemm_attr<pq::EPI_BF16, pq::ST_TMA_3D>()));
  PQ_TRY((gemm_attr<pq::EPI_GELU_BF16, pq::ST_REG>()));
  PQ_TRY((gemm_attr<pq::EPI_GELU_BF16, pq::ST_TMA_2D>()));
  PQ_TRY(set_smem(pq::gemm_bf16_lse_kernel, pq::GemmCfg::smem_bytes<false>()));
  PQ_TRY(set_smem(pq::gemm_bf16_topk_kernel, pq::GemmCfg::smem_bytes<false>()));
  PQ_TRY(set_smem(pq::tma_stream_bench_kernel, kTmaBenchSmem));
  int dev = 0, optin = 0;
  PQ_CUDA(cudaGetDevice(&dev));
  PQ_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  PQ_TRY(set_smem(pq::crop_resize_bicubic_kernel, static_cast<size_t>(optin)));   // sized per launch by the largest crop
  return PARSEQ_OK;
}

// init_kernel_attributes once per device: by parseq_create, and by the bare kernel exports, which may run without a handle
int ensure_kernel_attributes() {
  static std::mutex mu;
  static std::set<int> done;
  int dev = 0;
  PQ_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (done.count(dev) != 0) return PARSEQ_OK;
  PQ_TRY(init_kernel_attributes());
  done.insert(dev);
  return PARSEQ_OK;
}

// blocked_rows > 0: `out` is a column-blocked bf16 buffer [N/64][blocked_rows][64] (ptx.cuh: blocked_off); ldo is ignored
int gemm_launch(LaunchOpts& lo, const void* A, long long lda, const void* W, long long ldw, const float* bias, int M, int N,
                int K, int mode, float alpha, const float* resid, long long ldr, int resid_mod, void* out, long long ldo,
                cudaStream_t st, long long blocked_rows = 0) {
  if (M <= 0 || N <= 0 || K <= 0) return fail(PARSEQ_ERR_INVALID_ARG, "gemm: empty problem");
  if (mode != pq::EPI_F32 && mode != pq::EPI_BF16 && mode != pq::EPI_GELU_BF16)
    return fail(PARSEQ_ERR_INVALID_ARG, "gemm: mode must be 0 (fp32), 1 (bf16) or 2 (GELU bf16)");
  PQ_TRY(ensure_sm_count(lo));
  // One tile shape, 128 x 128, for every problem (the block_n / cta_group options are accepted and map onto it): QKV
  // (1152) and fc1 (1536) have no padded n-tile, and each ping-pong warpgroup holds one tile's accumulator.  Tiles are
  // numbered along N first, so the CTAs running at the same time share the rows of A they read (L2).
  CUtensorMap ta, tb, to;
  PQ_TRY(make_tmap(&ta, A, 2, M, K, lda, pq::GEMM_BLOCK_K, pq::GEMM_BLOCK_M));
  PQ_TRY(make_tmap(&tb, W, 2, N, K, ldw, pq::GEMM_BLOCK_K, pq::GEMM_BLOCK_N));
  pq::GemmParams p;
  p.M = M; p.N = N; p.K = K; p.alpha = alpha; p.bias = bias;
  p.resid = resid; p.ldr = ldr; p.resid_mod = resid_mod; p.out = out; p.ldo = ldo;
  const int esz = (mode == pq::EPI_F32) ? 4 : 2;
  bool vec = ((reinterpret_cast<uintptr_t>(out) & 7u) == 0) && ((ldo * esz) % 8 == 0);
  if (resid != nullptr) vec = vec && ((reinterpret_cast<uintptr_t>(resid) & 7u) == 0) && ((ldr * 4) % 8 == 0);
  p.vec_ok = vec ? 1 : 0;
  // bf16 tiles leave through a TMA store wherever the output is a valid tensor map (16-B aligned base and row pitch);
  // otherwise (e.g. a logits slice with an odd pitch) every thread stores its own values
  int store = pq::ST_REG;
  if (blocked_rows > 0) {
    if (mode != pq::EPI_BF16 || N % 64 != 0 || blocked_rows < M || (reinterpret_cast<uintptr_t>(out) & 15u) != 0)
      return fail(PARSEQ_ERR_INVALID_ARG, "gemm: blocked output needs a bf16 epilogue, N % 64 == 0 and rows >= M");
    // [N/64][blocked_rows][64] viewed as a 3D tensor of M rows per block: rows past M are never written
    PQ_TRY(make_tmap3d(&to, out, 64, M, N / 64, 64, 64 * blocked_rows, 64, pq::GEMM_BLOCK_M));
    store = pq::ST_TMA_3D;
  } else if (mode != pq::EPI_F32 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0 && (ldo * 2) % 16 == 0 && ldo >= N) {
    PQ_TRY(make_tmap(&to, out, 2, M, N, ldo, 64, pq::GEMM_BLOCK_M));
    store = pq::ST_TMA_2D;
  } else {
    to = ta;                                                  // unused by the register-store epilogues
  }
  p.max_stages = lo.gemm_stages;
  p.num_m_tiles = (M + pq::GEMM_BLOCK_M - 1) / pq::GEMM_BLOCK_M;
  p.num_n_tiles = (N + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  if (mode == pq::EPI_F32)
    return resid != nullptr ? launch_gemm_cfg<pq::EPI_F32_RESID, pq::ST_REG>(lo, ta, tb, to, p, tiles, st)
                            : launch_gemm_cfg<pq::EPI_F32, pq::ST_REG>(lo, ta, tb, to, p, tiles, st);
  if (mode == pq::EPI_BF16) {
    if (store == pq::ST_TMA_3D) return launch_gemm_cfg<pq::EPI_BF16, pq::ST_TMA_3D>(lo, ta, tb, to, p, tiles, st);
    return store == pq::ST_TMA_2D ? launch_gemm_cfg<pq::EPI_BF16, pq::ST_TMA_2D>(lo, ta, tb, to, p, tiles, st)
                                  : launch_gemm_cfg<pq::EPI_BF16, pq::ST_REG>(lo, ta, tb, to, p, tiles, st);
  }
  return store == pq::ST_TMA_2D ? launch_gemm_cfg<pq::EPI_GELU_BF16, pq::ST_TMA_2D>(lo, ta, tb, to, p, tiles, st)
                                : launch_gemm_cfg<pq::EPI_GELU_BF16, pq::ST_REG>(lo, ta, tb, to, p, tiles, st);
}

// The head GEMM with the log-sum-exp epilogue (gemm.cuh, gemm_bf16_lse_kernel): A[M, K] * W[N, K]^T + bias never leaves the registers;
// part[M][ceil(N / 128)] float2 per-tile (max, sum exp) partials, tlogit[row] = the logit of class tgt[row] (tgt may be
// null: partials only)
int gemm_lse_launch(LaunchOpts& lo, const void* A, long long lda, const void* W, long long ldw, const float* bias, int M, int N,
                    int K, const int* tgt, float2* part, float* tlogit, cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return fail(PARSEQ_ERR_INVALID_ARG, "gemm: empty problem");
  PQ_TRY(ensure_sm_count(lo));
  CUtensorMap ta, tb;
  PQ_TRY(make_tmap(&ta, A, 2, M, K, lda, pq::GEMM_BLOCK_K, pq::GEMM_BLOCK_M));
  PQ_TRY(make_tmap(&tb, W, 2, N, K, ldw, pq::GEMM_BLOCK_K, pq::GEMM_BLOCK_N));
  pq::GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.alpha = 1.0f; p.bias = bias;
  p.out = part;
  p.max_stages = lo.gemm_stages;
  p.num_m_tiles = (M + pq::GEMM_BLOCK_M - 1) / pq::GEMM_BLOCK_M;
  p.num_n_tiles = (N + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
  p.lse_tgt = tgt;
  p.lse_tlogit = tlogit;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  return launch_k(lo, pq::gemm_bf16_lse_kernel, dim3(static_cast<unsigned>(tiles < lo.sm_count ? tiles : lo.sm_count)),
                  dim3(pq::GEMM_THREADS), pq::GemmCfg::smem_bytes<false>(), st, ta, tb, ta, p);
}

// The head GEMM with the top-K epilogue (gemm.cuh, gemm_bf16_topk_kernel): per row and 128-column tile the (max, sum exp)
// partial of the allowed classes in part[M][ceil(N / 128)] and the tile's k best keys in keys[M][ceil(N / 128)][16];
// allowlist row of row r: mask + (r / mask_div) * ceil(N / 32), or no mask
int gemm_topk_launch(LaunchOpts& lo, const void* A, long long lda, const void* W, long long ldw, const float* bias, int M, int N,
                     int K, int k, const uint32_t* mask, int mask_div, float2* part, unsigned long long* keys, cudaStream_t st) {
  if (M <= 0 || N <= 0 || K <= 0) return fail(PARSEQ_ERR_INVALID_ARG, "gemm: empty problem");
  PQ_TRY(ensure_sm_count(lo));
  CUtensorMap ta, tb;
  PQ_TRY(make_tmap(&ta, A, 2, M, K, lda, pq::GEMM_BLOCK_K, pq::GEMM_BLOCK_M));
  PQ_TRY(make_tmap(&tb, W, 2, N, K, ldw, pq::GEMM_BLOCK_K, pq::GEMM_BLOCK_N));
  pq::GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.alpha = 1.0f; p.bias = bias;
  p.out = part;
  p.max_stages = lo.gemm_stages;
  p.num_m_tiles = (M + pq::GEMM_BLOCK_M - 1) / pq::GEMM_BLOCK_M;
  p.num_n_tiles = (N + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
  p.topk_keys = keys;
  p.topk_k = k;
  p.topk_mask = mask;
  p.topk_mask_div = mask_div;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  return launch_k(lo, pq::gemm_bf16_topk_kernel, dim3(static_cast<unsigned>(tiles < lo.sm_count ? tiles : lo.sm_count)),
                  dim3(pq::GEMM_THREADS), pq::GemmCfg::smem_bytes<false>(), st, ta, tb, ta, p);
}

// x[M, D] += A[M, K] * W[D, K]^T + bias (fp32, in place); xn[M, D] = bf16(LayerNorm(x; gamma, beta, eps))   (gemm_ln.cuh)
bool gemm_ln_supported(int D) { return D == 192 || D == 384; }
template <int D, int MODE>
int launch_gemm_ln(LaunchOpts& lo, const void* A, long long lda, const void* W, long long ldw, const float* bias, int M, int K, float* x,
                   const float* gamma, const float* beta, float eps, void* xn, cudaStream_t st) {
  using Cfg = pq::GemmLnCfg<D, MODE>;
  CUtensorMap ta, tb, tx;
  PQ_TRY(make_tmap(&ta, A, 2, M, K, lda, pq::GEMM_BLOCK_K, Cfg::kABox));
  PQ_TRY(make_tmap(&tb, W, 2, D, K, ldw, pq::GEMM_BLOCK_K, Cfg::kBox));
  if ((reinterpret_cast<uintptr_t>(x) & 7u) != 0 || (reinterpret_cast<uintptr_t>(xn) & 3u) != 0)
    return fail(PARSEQ_ERR_INVALID_ARG, "gemm_ln: x must be 8-byte and xn 4-byte aligned");
  pq::GemmLnParams p;
  p.M = M; p.K = K; p.bias = bias; p.gamma = gamma; p.beta = beta; p.eps = eps;
  p.num_m_tiles = (M + Cfg::kTileM - 1) / Cfg::kTileM;
  int clusters = p.num_m_tiles;
  if constexpr (MODE == 2) {
    // persistent: as many CTA pairs as the occupancy query admits on this device, each walking the tiles with the grid's
    // stride; x slices are fetched by TMA (x: 16-B aligned)
    PQ_TRY(make_tmap(&tx, x, 4, M, D, D, Cfg::kXBoxCols, pq::GLN_BLOCK_M));
    if (lo.ln_clusters == 0) {
      const LaunchConfig occ(dim3(static_cast<unsigned>(lo.sm_count / Cfg::kCG * Cfg::kCG)), dim3(pq::GLN_THREADS),
                             Cfg::kSmemBytes, st, Cfg::kCG, false);
      PQ_CUDA(cudaOccupancyMaxActiveClusters(&lo.ln_clusters, pq::gemm_ln_fused_kernel<D, MODE>, &occ.cfg));
      if (lo.ln_clusters <= 0) return fail(PARSEQ_ERR_CUDA, "gemm_ln: no cluster of the persistent kernel fits the device");
    }
    clusters = std::min(p.num_m_tiles, lo.ln_clusters);
  } else {
    tx = ta;                                                  // unused by MODE 0 / 1
  }
  return launch_ex(LaunchConfig(dim3(static_cast<unsigned>(clusters * Cfg::kCG)), dim3(pq::GLN_THREADS), Cfg::kSmemBytes, st,
                                Cfg::kCG, cluster_pdl(lo, Cfg::kCG)),
                   pq::gemm_ln_fused_kernel<D, MODE>, ta, tb, tx, x, reinterpret_cast<__nv_bfloat16*>(xn), p);
}
int gemm_ln_launch(LaunchOpts& lo, const void* A, long long lda, const void* W, long long ldw, const float* bias, int M, int D,
                   int K, float* x, const float* gamma, const float* beta, float eps, void* xn, cudaStream_t st) {
  if (M <= 0 || K <= 0) return fail(PARSEQ_ERR_INVALID_ARG, "gemm_ln: empty problem");
  PQ_TRY(ensure_sm_count(lo));
  PQ_TRY(load_driver_api());
  // MODE 2 (persistent CTA pairs on 64-row tiles, the columns split over the pair, ping-pong MMA warpgroups) runs every
  // K at D = 384: each tile's epilogue runs under the next tile's MMAs, and the residual arrives during the main loop.
  // ln_split: 0 auto (D = 384), 1 never (the full-row MODE 0 / MODE 1 kernel), 2 always.  The row statistics order is
  // chosen by K inside the kernel, never by the batch.  MODE 1 (ln_cta_group = 2 with ln_split = 1) shares the W tile
  // of two 64-row tiles by multicast.  Where the fused kernels are used at all is decided by the caller from the batch
  // regime (encode_chunk).
  if (D == 384 && lo.ln_split != 1)
    return launch_gemm_ln<384, 2>(lo, A, lda, W, ldw, bias, M, K, x, gamma, beta, eps, xn, st);
  if (lo.ln_cta_group == 2) {
    if (D == 384) return launch_gemm_ln<384, 1>(lo, A, lda, W, ldw, bias, M, K, x, gamma, beta, eps, xn, st);
    if (D == 192) return launch_gemm_ln<192, 1>(lo, A, lda, W, ldw, bias, M, K, x, gamma, beta, eps, xn, st);
  }
  if (D == 384) return launch_gemm_ln<384, 0>(lo, A, lda, W, ldw, bias, M, K, x, gamma, beta, eps, xn, st);
  if (D == 192) return launch_gemm_ln<192, 0>(lo, A, lda, W, ldw, bias, M, K, x, gamma, beta, eps, xn, st);
  return fail(PARSEQ_ERR_UNSUPPORTED, "gemm_ln: embed_dim must be 192 or 384");
}

// x[M, D] += GELU(xn W1^T + b1) W2^T + b2 (fp32, in place); xn_out = bf16(LayerNorm(x; gamma, beta, eps))   (mlp_ln.cuh)
template <int D, int CG>
int launch_mlp_ln(const LaunchOpts& lo, const void* xn, const void* W1, const float* b1, const void* W2, const float* b2, int M,
                  float* x, const float* gamma, const float* beta, float eps, void* xn_out, cudaStream_t st) {
  using Cfg = pq::MlpLnCfg<D, CG>;
  if ((reinterpret_cast<uintptr_t>(x) & 7u) != 0 || (reinterpret_cast<uintptr_t>(xn_out) & 3u) != 0)
    return fail(PARSEQ_ERR_INVALID_ARG, "mlp_ln: x must be 8-byte and xn_out 4-byte aligned");
  CUtensorMap txn, tw1, tw2;
  PQ_TRY(make_tmap(&txn, xn, 2, M, D, D, 64, pq::GLN_BLOCK_M));
  PQ_TRY(make_tmap(&tw1, W1, 2, Cfg::kH, D, D, 64, Cfg::kW1Rows));
  PQ_TRY(make_tmap(&tw2, W2, 2, D, Cfg::kH, Cfg::kH, 64, Cfg::kW2Rows));
  pq::MlpLnParams p;
  p.M = M; p.b1 = b1; p.b2 = b2; p.gamma = gamma; p.beta = beta; p.eps = eps;
  p.num_m_tiles = (M + pq::GLN_BLOCK_M * CG - 1) / (pq::GLN_BLOCK_M * CG);
  return launch_ex(LaunchConfig(dim3(static_cast<unsigned>(p.num_m_tiles * CG)), dim3(pq::MLP_THREADS), Cfg::kSmemBytes, st, CG,
                                cluster_pdl(lo, CG)),
                   pq::mlp_ln_fused_kernel<D, CG>, txn, tw1, tw2, x, reinterpret_cast<__nv_bfloat16*>(xn_out), p);
}
int mlp_ln_launch(LaunchOpts& lo, const void* xn, const void* W1, const float* b1, const void* W2, const float* b2, int M, int D,
                  float* x, const float* gamma, const float* beta, float eps, void* xn_out, cudaStream_t st) {
  if (M <= 0) return fail(PARSEQ_ERR_INVALID_ARG, "mlp_ln: empty problem");
  PQ_TRY(ensure_sm_count(lo));
  PQ_TRY(load_driver_api());
  // CTA pairs fetch every weight box once per 128 rows instead of 64 (multicast)
  const int CG = lo.mlp_cta_group ? lo.mlp_cta_group : 2;
  if (CG == 2) {
    if (D == 384) return launch_mlp_ln<384, 2>(lo, xn, W1, b1, W2, b2, M, x, gamma, beta, eps, xn_out, st);
    if (D == 192) return launch_mlp_ln<192, 2>(lo, xn, W1, b1, W2, b2, M, x, gamma, beta, eps, xn_out, st);
  }
  if (D == 384) return launch_mlp_ln<384, 1>(lo, xn, W1, b1, W2, b2, M, x, gamma, beta, eps, xn_out, st);
  if (D == 192) return launch_mlp_ln<192, 1>(lo, xn, W1, b1, W2, b2, M, x, gamma, beta, eps, xn_out, st);
  return fail(PARSEQ_ERR_UNSUPPORTED, "mlp_ln: embed_dim must be 192 or 384 (hidden width 4 * embed_dim)");
}

int layernorm_launch(const LaunchOpts& lo, const float* x, const float* g, const float* b, float eps, int M, int D, void* y, float* y32,
                     cudaStream_t st, const float* add = nullptr, int add_mod = 1, float* xw = nullptr) {
  const int rows_per_block = 8;
  const int grid = (M + rows_per_block - 1) / rows_per_block;
  __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y);
  switch (D) {
    case 192: return launch_k(lo, pq::layernorm_kernel<192>, dim3(grid), dim3(256), 0, st, x, g, b, eps, M, yb, y32, add, add_mod, xw);
    case 384: return launch_k(lo, pq::layernorm_kernel<384>, dim3(grid), dim3(256), 0, st, x, g, b, eps, M, yb, y32, add, add_mod, xw);
    case 768: return launch_k(lo, pq::layernorm_kernel<768>, dim3(grid), dim3(256), 0, st, x, g, b, eps, M, yb, y32, add, add_mod, xw);
    default: return fail(PARSEQ_ERR_UNSUPPORTED, "layernorm: embed_dim must be 192, 384 or 768");
  }
}

int enc_attention_launch(const LaunchOpts& lo, const void* qkv, int B, int T, int D, int heads, void* out, cudaStream_t st) {
  if (D != heads * pq::ATT_DH) return fail(PARSEQ_ERR_UNSUPPORTED, "encoder attention kernels cover head_dim=64");
  if (lo.attn_impl == 1 && T <= 256) {
    const dim3 grid(static_cast<unsigned>(B * heads), static_cast<unsigned>((T + 127) / 128));
    const __nv_bfloat16* q = reinterpret_cast<const __nv_bfloat16*>(qkv);
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    if (T <= 128)
      return launch_k(lo, pq::enc_attention_wgmma_kernel<128>, grid, dim3(pq::ATW_THREADS), pq::atw_smem_bytes<128>(), st, q, o, T, D, heads);
    return launch_k(lo, pq::enc_attention_wgmma_kernel<256>, grid, dim3(pq::ATW_THREADS), pq::atw_smem_bytes<256>(), st, q, o, T, D, heads);
  }
  if (T != pq::ATT_T) {   // masked two-pass mma.sync kernel, any token count
    return launch_k(lo, pq::enc_attention_any_kernel, dim3(B * heads, (T + pq::ATT_T - 1) / pq::ATT_T), dim3(256), 0, st,
                    reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(out), T, D, heads);
  }
  return launch_k(lo, pq::enc_attention_kernel, dim3(B * heads), dim3(256), 0, st,
                  reinterpret_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<__nv_bfloat16*>(out), D, heads);
}

// out[B*T, D] = attention(bf16(xn W_qkv^T + b_qkv)) in one kernel (qkv_attn.cuh): T = 128, head_dim 64, D in {192, 384}.
// Bit-identical to the QKV gemm (EPI_BF16) followed by enc_attention_launch with attn_impl = 0.
bool qkv_attn_supported(int T, int D, int heads) { return T == pq::ATT_T && D == heads * pq::ATT_DH && (D == 192 || D == 384); }
int qkv_attn_launch(LaunchOpts& lo, const void* xn, const void* W, const float* bias, int B, int T, int D, int heads, void* out,
                    cudaStream_t st) {
  if (B <= 0) return fail(PARSEQ_ERR_INVALID_ARG, "qkv_attn: empty batch");
  if (!qkv_attn_supported(T, D, heads))
    return fail(PARSEQ_ERR_UNSUPPORTED, "qkv_attn: T = 128, head_dim 64 and embed_dim 192 or 384 only");
  if ((reinterpret_cast<uintptr_t>(out) & 15u) != 0) return fail(PARSEQ_ERR_INVALID_ARG, "qkv_attn: out must be 16-byte aligned");
  PQ_TRY(ensure_sm_count(lo));
  CUtensorMap tx, tw;
  PQ_TRY(make_tmap(&tx, xn, 2, static_cast<long long>(B) * T, D, D, pq::GEMM_BLOCK_K, pq::ATT_T));
  PQ_TRY(make_tmap(&tw, W, 2, 3 * D, D, D, pq::GEMM_BLOCK_K, pq::ATT_DH));
  const int items = B * heads;
  const dim3 grid(static_cast<unsigned>(items < lo.sm_count ? items : lo.sm_count));   // persistent: one CTA per SM
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
  if (D == 192)
    return launch_k(lo, pq::enc_qkv_attn_kernel<192>, grid, dim3(pq::QA_THREADS), pq::QkvAttnCfg::kSmemBytes, st, tx, tw, bias, o, items);
  return launch_k(lo, pq::enc_qkv_attn_kernel<384>, grid, dim3(pq::QA_THREADS), pq::QkvAttnCfg::kSmemBytes, st, tx, tw, bias, o, items);
}

// The engine's streams are non-blocking, its events untimed (the timing events come from pool_event)
int make_stream(Stream* s) {
  cudaStream_t h = nullptr;
  PQ_CUDA(cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking));
  *s = Stream(h);
  return PARSEQ_OK;
}
int make_event(Event* ev) {
  cudaEvent_t h = nullptr;
  PQ_CUDA(cudaEventCreateWithFlags(&h, cudaEventDisableTiming));
  *ev = Event(h);
  return PARSEQ_OK;
}

struct Slot {
  std::string key;   // internal name (PARSeq state_dict key)
  std::string pub;   // state_dict key of the served architecture (== key for PARSeq; ViTSTR drops the "encoder." prefix)
  long long numel;
  bool bf16;
  DevBuf<unsigned char> dev;
  bool set;
};

// What the engine allocates for its sizes (max_batch, chunk, dec_chunk): the buffers alloc_workspace creates and those
// that calls reserve on first use.  A resize replaces all of it (free_workspace); the weights, the tables derived from
// them and the host-crop staging buffer stay.
struct Workspace {
  // encoder workspace (one pipeline stage = `chunk` images; the encoder runs serialised on `main`)
  DevBuf<__nv_bfloat16> a_pe, xn, qkv, att, hid;
  DevBuf<float> x;
  DevBuf<float> vt_rows;                            // ViTSTR tail: gathered token rows [chunk * L, D] fp32
  // per-stage decoder state: the decoder of stage s runs on its own stream while `main` encodes stage s+1
  DevBuf<__nv_bfloat16> mem, ckv;                   // [max_batch*T, D] encoder output, [max_batch*T, 2D] cross K/V
  std::vector<DevBuf<__nv_bfloat16>> ckv_deep;      // cross K/V of decoder layers 1..dec_depth-1, laid out as ckv
  // persistent AR-loop kernel state (whole super-chunk)
  DevBuf<__nv_bfloat16> ar_sa, ar_ca, ar_hd;
  DevBuf<float> ar_y, ar_qc, ar_part;
  DevBuf<int> ar_ids;               // [max_batch, ids_ld]
  DevBuf<unsigned int> ar_bar;
  DevBuf<unsigned long long> ar_prof;   // [32][16] phase time stamps of the AR kernel (debug option "ar_prof"; DESIGN.md 4)
  Event ev_enc;                     // `main`'s work so far, which the stage streams wait for (fan_out)
  struct Stage {
    DevBuf<__nv_bfloat16> sa, yn, ca, hd;
    DevBuf<float> y, qc;
    DevBuf<int> ids_ar, ids_ctx;    // [dec_chunk, ids_ld]
    // decoders of depth >= 2: content residual stream [dec_chunk * L, D] fp32, and the content K/V of layers
    // 1..dec_depth-1, one [dec_chunk, L, 2D] bf16 cache per layer (layer 0 reads the (position, token) table)
    DevBuf<float> cx;
    std::vector<DevBuf<__nv_bfloat16>> kvc;
    // candidate scoring (parseq_score), allocated by the first score call: per-tile log-sum-exp partials
    // [dec_chunk * L][ceil(C / 128)] and target logits of the chain's rows
    DevBuf<float2> lse_part;
    DevBuf<float> lse_tlogit;
    // beam search (parseq_beam_search), allocated by the first beam call: double-buffered state of `rows` beam rows
    // (ids [rows][ids_ld], score, len, st; kernels.cuh beam_select_kernel), the parent row of each new beam, what the
    // head leaves of one step's rows (ViTSTR: of `rows / BEAM_MAX` images' positions) - the logits at <= 128 classes, the
    // top-K epilogue's partials and keys above - and at depth >= 2 a second content K/V cache per layer that the parents'
    // rows are gathered into
    struct Beam {
      int rows = 0;
      DevBuf<int> ids[2];
      DevBuf<float> score[2];
      DevBuf<int> len[2];
      DevBuf<int> st[2];
      DevBuf<int> parent;
      DevBuf<float> logits;              // <= 128 classes: the step's logits
      DevBuf<float2> part;               // > 128 classes: the top-K epilogue's LSE partials [lrows][ceil(C / 128)]
      DevBuf<unsigned long long> keys;   //   and keys [lrows][ceil(C / 128)][BEAM_TOPK_LD]
      std::vector<DevBuf<__nv_bfloat16>> kvc;
      // lexicon search (parseq_beam_search_lexicon), allocated by the first lexicon call: each beam row's lexicon node,
      // double-buffered; above 128 classes `logits` is allocated then as well (the lexicon step reads whole rows)
      DevBuf<int> node[2];
    } bm;
    Stream stream;
    Event ev_done;
  };
  std::vector<Stage> stages;
  // static I/O buffers the CUDA graphs are captured on
  DevBuf<float> in_images, out_logits;
  DevBuf<int> out_ids, out_steps;
  DevBuf<float> out_maps;           // [max_batch, L, T] cross-attention maps, allocated by the first call that asks for them
  DevBuf<uint8_t> in_images_u8;     // static input of the uint8 HWC entry points
  DevBuf<uint32_t> in_mask;         // [max_batch, mask_ld] class allowlist rows of the super-chunk (graphs, host entry points)
  DevBuf<pq::CropDesc> crop_tab;    // the resize kernel's crop table [max_batch] (raw-crop entry points, crops.cuh)
  DevBuf<pq::RegionDesc> reg_tab;   // the warp kernel's region table [max_batch], allocated by the first parseq_warp_regions
  DevBuf<pq::TpsDesc> tps_tab;      // the TPS kernel's polygon table [max_batch], allocated by the first parseq_warp_polygons
  // candidate scoring: the call's metadata (ids, targets, row tables; grown on demand), one causal [P][P] mask per
  // P = 1..L (mask of P at sc_causal + (P - 1) * L * L), and ViTSTR's LSE partials of a chunk's (image, position) rows
  DevBuf<int> sc_meta;
  DevBuf<unsigned char> sc_causal;
  DevBuf<float2> sc_vt_part;
  long long beam_bytes = 0;         // device bytes of the beam-search buffers (0 until the first beam call)
  DevBuf<int> lex_roots;            // the lexicon call's roots (grown on demand)
  // orientation search (parseq_forward_crops_oriented), allocated by the first oriented call: the crop of each pass-2
  // reading of a super-chunk [max_batch], the readings' confidences [max_batch], and the running step count of the call
  DevBuf<int> or_rd, or_steps;
  DevBuf<float> or_conf;
};

}  // namespace

// The engine derives from its workspace so that the call sites name its buffers directly (e->x, e->stages).  Its own
// members are destroyed before the workspace base, and `graphs` before every other member: the graphs go before the
// buffers they captured.
struct parseq_engine : Workspace {
  parseq_config cfg;
  int D, T, Kp, Me, Md, L, V, C, gh, gw, dh_dec;   // T: tokens per image in the encoder (patches + class token if any)
  int ids_ld = 32;                                   // row pitch of the decoder's id buffers: 32 (L <= 32) or 64 (L <= 64)
  int arch = 0, Tp = 0;                              // arch 1 = ViTSTR; Tp = gh * gw patches
  std::map<std::string, int> pub_index;
  int chunk;
  std::vector<Slot> slots;
  std::map<std::string, int> index;
  bool finalized = false;
  bool broken = false;                               // workspace could not be (re)allocated: every forward fails
  LaunchOpts lo;                                     // per-handle launch options
  long long launches = 0;
  // optional per-category device timing (bench.py roofline pass; off on the throughput pass)
  bool timing = false;
  struct TimedLaunch { int cat; double flops; Event a, b; };
  std::vector<TimedLaunch> timed;
  std::vector<Event> event_pool;
  int cur_cat = 5;
  // derived tables
  DevBuf<__nv_bfloat16> kvtab;      // [L*V, 2D]
  DevBuf<float> qs;                 // [L, D]
  int dec_chunk = 128;              // images per decoder chain (each chain runs on its own stream)
  // persistent AR-loop kernel state (whole super-chunk)
  int ar_kernel = 2;                // option "ar_kernel": 0 chain, 1 grid-barrier kernel, 2 cluster kernel where it applies (ar_path)
  pq::DecAr2Maps ar2_maps[2];       // TMA descriptors (decoder weights, K/V cache) for cluster size 8 [0] and 6 [1]
  bool ar2_maps_ok = false;
  int ar2_clusters[3][2] = {{0, 0}, {0, 0}, {0, 0}};   // max co-resident clusters, index [MT][cluster size 6 ? 1 : 0]
  int ar2_occ[3][2] = {{0, 0}, {0, 0}, {0, 0}};        // what cudaOccupancyMaxActiveClusters answered (debug)
  int ar_last_cs = 0;
  int ar_last_per = 0, ar_last_ncl = 0;
  int ar_last_mt = 0, ar_last_hs = 0, ar_last_wide = 0, ar_last_idp = 0;   // last cluster-kernel instantiation (debug)
  int ar_last_path = -1;            // AR loop of the last forward: ArPath (0 chain, 1 grid barrier, 2 cluster), -1 none (debug)
  int ar_cs = 0;                    // option "ar_cluster_size": 0 = auto, 6 / 8 = forced
  int ar_clusters_override = 0;     // option "ar_clusters": clusters the AR kernel spreads a batch over (0 = derived)
  int fuse_mlp = 0;                 // fc1 + GELU + fc2 + residual + LayerNorm in one kernel (mlp_ln.cuh) where fuse_ln bit 1 applies
  int fuse_ln = 3;                  // bit 0: attn.proj, bit 1: mlp.fc2 also produce the LayerNorm that follows (gemm_ln.cuh)
  bool ar_prof_on = false;
  int max_batch = 512;              // images per graph / super-chunk = stages.size() * chunk
  Stream main;                      // engine-owned: user stream -> (event) -> main -> (event) -> user stream
  Stream copy;                      // host entry points: input upload in two halves, overlapped with the first half's encoder
  Event ev_c[3];
  Event ev_in, ev_out;
  int mask_ld = 0;                  // words per allowlist row: ceil(C / 32)
  // raw-crop entry points (crops.cuh): the host copy of the crop table of the current super-chunk, and the device copy
  // of a super-chunk's packed bytes for the host entry point (grown on demand)
  std::vector<pq::CropDesc> crop_descs;
  long long crop_base = 0;
  std::vector<pq::RegionDesc> reg_descs;   // parseq_warp_regions: the host copy of a chunk's region table (regions.cuh)
  std::vector<pq::TpsDesc> tps_descs;      // parseq_warp_polygons: the host copy of a chunk's polygon table
  DevBuf<uint8_t> crop_stage;
  bool use_graph = true;
  long long orient_rereads = 0, orient_readings = 0;   // pass 2 of the last oriented call: crops re-read, readings run
  struct GraphEntry { GraphExec exec; long long kernels; };
  std::map<std::vector<int>, GraphEntry> graphs;   // last member: destroyed first

  void* w(const std::string& k) const { return slots[index.at(k)].dev; }
  const float* wf(const std::string& k) const { return reinterpret_cast<const float*>(w(k)); }
  const __nv_bfloat16* wb(const std::string& k) const { return reinterpret_cast<const __nv_bfloat16*>(w(k)); }
};

// A lexicon DAG on one device (parseq_lexicon_create): the CSR arrays of parseq_lexicon_desc
struct parseq_lexicon {
  int device = 0, C = 0, V = 0, E = 0;
  DevBuf<int> first_edge;           // [V + 1]
  DevBuf<int> edge_class;           // [max(E, 1)]
  DevBuf<int> edge_child;           // [max(E, 1)]
  DevBuf<unsigned char> terminal;   // [V]
};

template <typename T>
int DevBuf<T>::alloc(long long n) {
  reset();
  void* p = nullptr;
  PQ_CUDA(cudaMalloc(&p, static_cast<size_t>(n) * sizeof(T)));
  p_ = static_cast<T*>(p);
  n_ = n;
  g_live_bytes += bytes();
  return PARSEQ_OK;
}

template <typename T>
int DevBuf<T>::grow(const parseq_engine* e, long long n) {
  if (n <= n_) return PARSEQ_OK;
  if (p_ != nullptr) {
    PQ_CUDA(cudaStreamSynchronize(e->main));
    PQ_CUDA(cudaStreamSynchronize(e->copy));
  }
  return alloc(n);
}

namespace {

void add_slot(parseq_engine* e, const std::string& key, long long numel, bool bf16) {
  std::string pub = key;
  if (e->arch == 1 && key.rfind("encoder.", 0) == 0) pub = key.substr(8);
  e->index[key] = static_cast<int>(e->slots.size());
  e->pub_index[pub] = static_cast<int>(e->slots.size());
  e->slots.push_back(Slot{key, pub, numel, bf16, {}, false});
}

// The handle can run a call: not null, its workspace allocated, and (`weights`) its weights finalized.
int check_ready(const parseq_engine* e, bool weights = true) {
  if (e == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (e->broken) return fail(PARSEQ_ERR_STATE, "engine workspace is gone (a failed resize): destroy the handle");
  if (weights && !e->finalized)
    return fail(PARSEQ_ERR_STATE, "parseq_finalize has not been called after the last weight update");
  return PARSEQ_OK;
}

// The stream bracket of an entry point: the engine's work runs on `main` after what the caller enqueued on `user`
// before the call (enter_main), and the caller's later work runs after it (leave_main; not reached on an error).
int enter_main(parseq_engine* e, cudaStream_t user) {
  PQ_CUDA(cudaEventRecord(e->ev_in, user));
  PQ_CUDA(cudaStreamWaitEvent(e->main, e->ev_in, 0));
  return PARSEQ_OK;
}
int leave_main(parseq_engine* e, cudaStream_t user) {
  PQ_CUDA(cudaEventRecord(e->ev_out, e->main));
  PQ_CUDA(cudaStreamWaitEvent(user, e->ev_out, 0));
  return PARSEQ_OK;
}

// Bytes per input image: fp32 NCHW or uint8 HWC
long long image_bytes(const parseq_engine* e, bool u8) { return 3ll * e->cfg.img_h * e->cfg.img_w * (u8 ? 1 : 4); }

int alloc_workspace(parseq_engine* e) {
  const long long R = static_cast<long long>(e->chunk) * e->T;          // encoder rows per chunk
  const long long RB = static_cast<long long>(e->max_batch) * e->T;     // rows of a whole super-chunk
  const long long Rd = static_cast<long long>(e->dec_chunk) * e->L;     // decoder rows per chain
  const int D = e->D;
  PQ_TRY(e->a_pe.alloc(R * e->Kp));
  PQ_TRY(e->x.alloc(R * D));
  PQ_TRY(e->xn.alloc(R * D));
  PQ_TRY(e->qkv.alloc(R * 3 * D));
  PQ_TRY(e->att.alloc(R * D));
  PQ_TRY(e->hid.alloc(R * e->Me));
  PQ_TRY(e->mem.alloc(RB * D));
  PQ_TRY(e->ckv.alloc(RB * 2 * D));
  if (e->cfg.dec_depth > 1) {
    e->ckv_deep.resize(static_cast<size_t>(e->cfg.dec_depth - 1));
    for (auto& c : e->ckv_deep) PQ_TRY(c.alloc(RB * 2 * D));
  }
  PQ_TRY(e->ar_sa.alloc(1ll * e->max_batch * D));
  PQ_TRY(e->ar_ca.alloc(1ll * e->max_batch * D));
  PQ_TRY(e->ar_hd.alloc(1ll * e->max_batch * e->Md));
  PQ_TRY(e->ar_y.alloc(1ll * e->max_batch * D));
  PQ_TRY(e->ar_qc.alloc(1ll * e->max_batch * D));
  PQ_TRY(e->ar_part.alloc(3ll * e->max_batch * D));
  PQ_TRY(e->ar_ids.alloc(1ll * e->max_batch * e->ids_ld));
  PQ_TRY(e->ar_bar.alloc(64));
  PQ_TRY(e->ar_prof.alloc(32 * 16));
  if (e->arch == 1) PQ_TRY(e->vt_rows.alloc(1ll * e->chunk * e->L * D));
  PQ_TRY(make_event(&e->ev_enc));
  const int n_stages = (e->max_batch + e->dec_chunk - 1) / e->dec_chunk;
  e->stages.resize(static_cast<size_t>(n_stages));
  for (auto& sg : e->stages) {
    PQ_TRY(sg.sa.alloc(Rd * D));
    PQ_TRY(sg.yn.alloc(Rd * D));
    PQ_TRY(sg.ca.alloc(Rd * D));
    PQ_TRY(sg.hd.alloc(Rd * e->Md));
    PQ_TRY(sg.y.alloc(Rd * D));
    PQ_TRY(sg.qc.alloc(Rd * D));
    PQ_TRY(sg.ids_ar.alloc(static_cast<long long>(e->dec_chunk) * e->ids_ld));
    PQ_TRY(sg.ids_ctx.alloc(static_cast<long long>(e->dec_chunk) * e->ids_ld));
    if (e->cfg.dec_depth > 1) {
      PQ_TRY(sg.cx.alloc(Rd * D));
      sg.kvc.resize(static_cast<size_t>(e->cfg.dec_depth - 1));
      for (auto& c : sg.kvc) PQ_TRY(c.alloc(Rd * 2 * D));
    }
    PQ_TRY(make_stream(&sg.stream));
    PQ_TRY(make_event(&sg.ev_done));
  }
  const long long NB = e->max_batch;
  PQ_TRY(e->in_images.alloc(NB * 3 * e->cfg.img_h * e->cfg.img_w));
  PQ_TRY(e->in_images_u8.alloc(NB * 3 * e->cfg.img_h * e->cfg.img_w));
  PQ_TRY(e->crop_tab.alloc(NB));
  PQ_TRY(e->in_mask.alloc(NB * e->mask_ld));
  PQ_TRY(e->out_logits.alloc(NB * e->L * e->C));
  PQ_TRY(e->out_ids.alloc(NB * e->L));
  PQ_TRY(e->out_steps.alloc(4));
  return PARSEQ_OK;
}

// Back to no workspace: the graphs first (they captured its buffers), and the cluster AR kernel's tensor maps, which hold
// the address of the K/V cache.
void free_workspace(parseq_engine* e) {
  e->graphs.clear();
  e->ar2_maps_ok = false;
  static_cast<Workspace&>(*e) = Workspace();
}

// categories: 0 encoder GEMM, 1 encoder attention, 2 LayerNorm, 3 decoder GEMM, 4 decoder attention, 5 other,
// 6 encoder residual GEMM + LayerNorm, 7 AR-loop kernel, 8 scoring tail (head GEMM with the LSE epilogue + reduce),
// 9 beam selection (beam_select_kernel and the K/V gather of parseq_beam_search), 10 cross-attention maps
// (dec_cross_attn_maps_kernel, its grouped form, maps_zero_tail_kernel), 11 orientation search (orient.cuh:
// confidence, select, pass-2 allowlist gather)
enum { CAT_ENC_GEMM = 0, CAT_ENC_ATTN = 1, CAT_LN = 2, CAT_DEC_GEMM = 3, CAT_DEC_ATTN = 4, CAT_MISC = 5, CAT_ENC_GEMM_LN = 6, CAT_DEC_AR = 7,
       CAT_SCORE = 8, CAT_BEAM = 9, CAT_MAPS = 10, CAT_ORIENT = 11, CAT_COUNT = 12 };

Event pool_event(parseq_engine* e) {
  if (!e->event_pool.empty()) { Event ev = std::move(e->event_pool.back()); e->event_pool.pop_back(); return ev; }
  cudaEvent_t ev = nullptr; cudaEventCreate(&ev); return Event(ev);
}
struct TimedScope {   // records a CUDA-event pair around the launches issued in its lifetime
  parseq_engine* e; cudaStream_t st; int idx = -1;
  TimedScope(parseq_engine* e_, cudaStream_t st_, int cat, double flops) : e(e_), st(st_) {
    e->launches++;
    if (!e->timing) return;
    parseq_engine::TimedLaunch t{cat, flops, pool_event(e), pool_event(e)};
    cudaEventRecord(t.a, st);
    e->timed.push_back(std::move(t));
    idx = static_cast<int>(e->timed.size()) - 1;
  }
  ~TimedScope() { if (idx >= 0) cudaEventRecord(e->timed[idx].b, st); }
};

int gemm(parseq_engine* e, const void* A, long long lda, const void* W, long long ldw, const float* bias, int M, int N,
         int K, int mode, float alpha, const float* resid, long long ldr, int resid_mod, void* out, long long ldo,
         cudaStream_t st, long long blocked_rows = 0) {
  TimedScope ts(e, st, e->cur_cat == CAT_DEC_GEMM ? CAT_DEC_GEMM : CAT_ENC_GEMM, 2.0 * M * N * K);
  return gemm_launch(e->lo, A, lda, W, ldw, bias, M, N, K, mode, alpha, resid, ldr, resid_mod, out, ldo, st, blocked_rows);
}
// x += A W^T + b;  y = bf16(LayerNorm(x; <ln_prefix>))  in one kernel
int gemm_ln(parseq_engine* e, const void* A, long long lda, const std::string& lin, int M, int K, float* x,
            const std::string& ln_prefix, float eps, void* y, cudaStream_t st) {
  TimedScope ts(e, st, CAT_ENC_GEMM_LN, 2.0 * M * e->D * K);
  return gemm_ln_launch(e->lo, A, lda, e->w(lin + ".weight"), K, e->wf(lin + ".bias"), M, e->D, K, x, e->wf(ln_prefix + ".weight"),
                        e->wf(ln_prefix + ".bias"), eps, y, st);
}
// x += fc2(GELU(fc1(xn)));  y = bf16(LayerNorm(x; <ln_prefix>))  in one kernel (block prefix `blk`, e.g. "encoder.blocks.3.")
int mlp_ln(parseq_engine* e, const void* xn, const std::string& blk, int M, float* x, const std::string& ln_prefix, float eps,
           void* y, cudaStream_t st) {
  TimedScope ts(e, st, CAT_ENC_GEMM_LN, 4.0 * M * e->D * e->Me);
  return mlp_ln_launch(e->lo, xn, e->w(blk + "mlp.fc1.weight"), e->wf(blk + "mlp.fc1.bias"), e->w(blk + "mlp.fc2.weight"),
                       e->wf(blk + "mlp.fc2.bias"), M, e->D, x, e->wf(ln_prefix + ".weight"), e->wf(ln_prefix + ".bias"), eps, y, st);
}
int layernorm(parseq_engine* e, const float* x, const std::string& prefix, float eps, int M, void* y, float* y32,
              cudaStream_t st, const float* add = nullptr, int add_mod = 1, float* xw = nullptr) {
  TimedScope ts(e, st, CAT_LN, 0.0);
  return layernorm_launch(e->lo, x, e->wf(prefix + ".weight"), e->wf(prefix + ".bias"), eps, M, e->D, y, y32, st, add, add_mod, xw);
}

// ---------------------------------------------------------------- encoder (model.py:83-84 -> timm forward_features)
int encode_chunk(parseq_engine* e, const void* images_any, bool u8, int B, __nv_bfloat16* mem_out, float* memory32,
                 cudaStream_t st, bool final_norm = true, int regime_batch = 0) {
  // regime_batch: the batch whose size selects the kernel variants (a half batch encoded on its own, under the upload of
  // the other half, must run the kernels the whole batch would: rows stay bit-identical to the unsplit call)
  const int D = e->D, T = e->T, M = B * T;
  e->cur_cat = CAT_ENC_GEMM;
  {
    TimedScope ts(e, st, CAT_MISC, 0.0);
    if (u8) {
      const long long total = static_cast<long long>(B) * e->gh * e->gw * e->cfg.patch_h;
      const int grid = static_cast<int>((total + 255) / 256);
      PQ_TRY(launch_k(e->lo, pq::im2col_patch_u8_kernel, dim3(grid), dim3(256), 0, st, static_cast<const uint8_t*>(images_any), e->a_pe,
                      B, e->cfg.img_h, e->cfg.img_w, e->cfg.patch_h, e->cfg.patch_w, e->gh, e->gw));
    } else {
      const long long total = static_cast<long long>(B) * e->gh * e->gw * 3 * e->cfg.patch_h;
      const int grid = static_cast<int>((total + 255) / 256);
      PQ_TRY(launch_k(e->lo, pq::im2col_patch_kernel, dim3(grid), dim3(256), 0, st, static_cast<const float*>(images_any), e->a_pe, B,
                      e->cfg.img_h, e->cfg.img_w, e->cfg.patch_h, e->cfg.patch_w, e->gh, e->gw));
    }
  }
  if (e->arch == 0) {
    // x = patches * Wpe^T + bpe + pos_embed
    PQ_TRY(gemm(e, e->a_pe, e->Kp, e->w("encoder.patch_embed.proj.weight"), e->Kp,
                e->wf("encoder.patch_embed.proj.bias"), M, D, e->Kp, pq::EPI_F32, 1.0f, e->wf("encoder.pos_embed"), D, T,
                e->x, D, st));
  } else {
    // timm _pos_embed with a class token: x = cat(cls_token, patches * Wpe^T + bpe) + pos_embed[0..Tp]
    float* tmp = reinterpret_cast<float*>(e->hid.get());      // [B*Tp, D] fp32 fits the (still unused) [B*T, 4D] bf16 MLP buffer
    PQ_TRY(gemm(e, e->a_pe, e->Kp, e->w("encoder.patch_embed.proj.weight"), e->Kp,
                e->wf("encoder.patch_embed.proj.bias"), B * e->Tp, D, e->Kp, pq::EPI_F32, 1.0f,
                e->wf("encoder.pos_embed") + D, D, e->Tp, tmp, D, st));
    TimedScope ts(e, st, CAT_MISC, 0.0);
    const long long total = 1ll * M * (D / 4);
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 132ll * 16));
    PQ_TRY(launch_k(e->lo, pq::cls_assemble_kernel, dim3(grid), dim3(256), 0, st, reinterpret_cast<const float4*>(tmp),
                    reinterpret_cast<const float4*>(e->wf("encoder.cls_token")),
                    reinterpret_cast<const float4*>(e->wf("encoder.pos_embed")), reinterpret_cast<float4*>(e->x.get()), B, e->Tp,
                    D / 4));
  }
  // With fuse_ln the two residual GEMMs of a block also emit the LayerNorm that consumes their result (norm2 after
  // attn.proj; the next block's norm1 - or the final encoder.norm - after mlp.fc2): the fp32 residual stream is read
  // and written once per GEMM instead of once more per LayerNorm.
  // The fused kernel owns whole rows (the columns of a row are not spread over tiles): it is used once the 128-row
  // tiles fill the machine about twice; below that the N-split GEMM + LayerNorm pair has more CTAs to spread over the
  // SMs.  "fuse_ln" bit 2 forces it for any M (tests).
  const int Mr = (regime_batch > B ? regime_batch : B) * T;
  const bool big = (Mr + pq::GEMM_BLOCK_M - 1) / pq::GEMM_BLOCK_M >= 2 * e->lo.sm_count || (e->fuse_ln & 4);
  const bool fuse_proj = (e->fuse_ln & 1) && gemm_ln_supported(D) && big;
  const bool fuse_fc2 = (e->fuse_ln & 2) && gemm_ln_supported(D) && big;
  const bool fuse_mlp = e->fuse_mlp && fuse_fc2 && e->Me == 4 * D;
  // QKV + attention in one kernel wherever it applies (bit-identical to the pair, so at every batch size); the wgmma
  // attention (attn_impl = 1) and the other token counts keep the QKV GEMM + attention kernel pair
  const bool fuse_qkv_attn = e->lo.attn_impl == 0 && qkv_attn_supported(T, D, e->cfg.enc_num_heads);
  bool final_done = false;
  for (int i = 0; i < e->cfg.enc_depth; ++i) {
    const std::string p = "encoder.blocks." + std::to_string(i) + ".";
    const bool last = (i == e->cfg.enc_depth - 1);
    if (!(fuse_fc2 && i > 0)) PQ_TRY(layernorm(e, e->x, p + "norm1", 1e-6f, M, e->xn, nullptr, st));
    if (fuse_qkv_attn) {
      // the QKV projection and the attention core in one kernel: qkv stays on the SM
      TimedScope ts(e, st, CAT_ENC_GEMM, 2.0 * M * 3 * D * D + 4.0 * B * T * T * D);
      PQ_TRY(qkv_attn_launch(e->lo, e->xn, e->w(p + "attn.qkv.weight"), e->wf(p + "attn.qkv.bias"), B, T, D,
                             e->cfg.enc_num_heads, e->att, st));
    } else {
      PQ_TRY(gemm(e, e->xn, D, e->w(p + "attn.qkv.weight"), D, e->wf(p + "attn.qkv.bias"), M, 3 * D, D, pq::EPI_BF16,
                  1.0f, nullptr, 0, 0, e->qkv, 3 * D, st));
      TimedScope ts(e, st, CAT_ENC_ATTN, 4.0 * B * T * T * D);
      PQ_TRY(enc_attention_launch(e->lo, e->qkv, B, T, D, e->cfg.enc_num_heads, e->att, st));
    }
    if (fuse_proj) {
      PQ_TRY(gemm_ln(e, e->att, D, p + "attn.proj", M, D, e->x, p + "norm2", 1e-6f, e->xn, st));
    } else {
      PQ_TRY(gemm(e, e->att, D, e->w(p + "attn.proj.weight"), D, e->wf(p + "attn.proj.bias"), M, D, D, pq::EPI_F32, 1.0f,
                  e->x, D, 0, e->x, D, st));
      PQ_TRY(layernorm(e, e->x, p + "norm2", 1e-6f, M, e->xn, nullptr, st));
    }
    if (fuse_mlp && (!last || (final_norm && memory32 == nullptr))) {
      // the whole MLP + the next LayerNorm in one kernel: the hidden activation never leaves the SM (mlp_ln.cuh)
      if (!last) {
        PQ_TRY(mlp_ln(e, e->xn, p, M, e->x, "encoder.blocks." + std::to_string(i + 1) + ".norm1", 1e-6f, e->xn, st));
      } else {
        PQ_TRY(mlp_ln(e, e->xn, p, M, e->x, "encoder.norm", 1e-6f, mem_out, st));
        final_done = true;
      }
      continue;
    }
    PQ_TRY(gemm(e, e->xn, D, e->w(p + "mlp.fc1.weight"), D, e->wf(p + "mlp.fc1.bias"), M, e->Me, D, pq::EPI_GELU_BF16,
                1.0f, nullptr, 0, 0, e->hid, e->Me, st));
    if (fuse_fc2 && !last) {
      PQ_TRY(gemm_ln(e, e->hid, e->Me, p + "mlp.fc2", M, e->Me, e->x, "encoder.blocks." + std::to_string(i + 1) + ".norm1",
                     1e-6f, e->xn, st));
    } else if (fuse_fc2 && final_norm && memory32 == nullptr) {
      PQ_TRY(gemm_ln(e, e->hid, e->Me, p + "mlp.fc2", M, e->Me, e->x, "encoder.norm", 1e-6f, mem_out, st));
      final_done = true;
    } else {
      PQ_TRY(gemm(e, e->hid, e->Me, e->w(p + "mlp.fc2.weight"), e->Me, e->wf(p + "mlp.fc2.bias"), M, D, e->Me,
                  pq::EPI_F32, 1.0f, e->x, D, 0, e->x, D, st));
    }
  }
  if (final_done) return PARSEQ_OK;
  if (final_norm) PQ_TRY(layernorm(e, e->x, "encoder.norm", 1e-6f, M, mem_out, memory32, st));
  return PARSEQ_OK;
}

// ---------------------------------------------------------------- ViTSTR tail (vitstr/model.py:19-28, vitstr/system.py:65-71)
// logits[b, j] = head(norm(x[b, 1 + j])), j < L = max_length + 1: the reference computes tokens [0, max_length + 2) and
// drops token 0 (the class token); norm and head are row-wise, so only the kept rows are gathered and computed.
int argmax_rows(parseq_engine* e, float* logits, int L, int B, int nrows, int src0, int* ids, int ids_ld, int dst0,
                const int* forced, int forced_ld, const uint32_t* mask, cudaStream_t st);
// e->xn [B * L, D] = bf16(norm(x[b, 1 + j])), j < L: the rows the head reads
int vitstr_rows(parseq_engine* e, int B, int L, cudaStream_t st) {
  const int D = e->D, M = B * L;
  {
    TimedScope ts(e, st, CAT_MISC, 0.0);
    const long long total = 1ll * M * (D / 4);
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 132ll * 16));
    PQ_TRY(launch_k(e->lo, pq::gather_token_rows_kernel, dim3(grid), dim3(256), 0, st, reinterpret_cast<const float4*>(e->x.get()),
                    reinterpret_cast<float4*>(e->vt_rows.get()), B, e->T, 1, L, D / 4));
  }
  return layernorm(e, e->vt_rows, "encoder.norm", 1e-6f, M, e->xn, nullptr, st);
}
int vitstr_tail(parseq_engine* e, int B, int L, float* logits, int* ids_out, const uint32_t* mask, cudaStream_t st) {
  const int D = e->D, M = B * L;
  PQ_TRY(vitstr_rows(e, B, L, st));
  PQ_TRY(gemm(e, e->xn, D, e->w("head.weight"), D, e->wf("head.bias"), M, e->C, D, pq::EPI_F32, 1.0f, nullptr, 0, 0, logits,
              e->C, st));
  // vitstr/model.py:26 applies the head to [B * s, D] rows: row r belongs to image r / s, the allowlist row it takes
  if (ids_out != nullptr || mask != nullptr) PQ_TRY(argmax_rows(e, logits, L, B, L, 0, ids_out, L, 0, nullptr, 0, mask, st));
  return PARSEQ_OK;
}

// ---------------------------------------------------------------- one Decoder call (model.py:86-103, modules.py:55-125)
// The self-attention mask (the int the kernels take): keys 0..nkeys-1 (AR step, NAR), the cloze mask + first EOS
// (refinement), or the caller's masks over one query row per (image, query) (PARSeq.decode), which only self_mask picks.
enum class SelfMask : int { Keys = 0, Cloze = 1, Caller = 2 };
// What a pass ends with after the last layer: decoder.norm, then the head into logits (+ greedy ids), the head GEMM's
// LSE or top-K epilogue (no logits stored), or nothing more (Norm); or it stops after the last layer's maps (MapsOnly:
// no cross-attention output, MLP or decoder.norm)
enum class Tail { Head, LogSumExp, TopK, Norm, MapsOnly };

// One decoder pass: rows (b, qi), qi in [0, nq), of images b_first.. of the super-chunk (rows of the cross K/V cache);
// query position q0 + qi; context ids[b, 0..nkeys-1] (id rows [B, ids_ld]).  Callers assign the fields they use.
struct DecodePass {
  int b_first = 0, B = 0, nq = 0, q0 = 0, nkeys = 0;
  const int* ids = nullptr;
  // an AR step (nq = 1, keys 0..q0): the content stream computes row q0 only and appends it to the caches of pitch L;
  // otherwise it computes the whole context (nkeys rows per image, pitch nkeys)
  bool ar_step = false;
  int kv_pitch(const parseq_engine* e) const { return ar_step ? e->L : nkeys; }
  int beam = 1;                          // beam search: B counts beam rows, `beam` consecutive rows per image; the rows'
                                         // self-attention reads their own ids, their cross-attention their image
  SelfMask self_mask = SelfMask::Keys;
  // caller inputs of PARSeq.decode (model.py:86-103) that the inference loops never use
  const float* query = nullptr;          // [B*nq, D] fp32 raw queries (residual base); null -> pos_queries[q0 + qi]
  const unsigned char* qmask = nullptr;  // [nq, nkeys], 1 = masked
  const unsigned char* pmask = nullptr;  // [B, nkeys], 1 = masked
  const unsigned char* cmask = nullptr;  // [nkeys, nkeys] content-stream mask (`tgt_mask`), 1 = masked; depth >= 2 only
  // candidate scoring: the B rows are candidates of cand_imgs images, image j's candidates [cand_off[j], cand_off[j + 1])
  // (device), at most cand_max_rows query rows per image; every cross-attention of the pass serves a candidate's rows
  // from its image (dec_cross_attn3_grouped_kernel)
  const int* cand_off = nullptr;
  int cand_imgs = 0, cand_max_rows = 0;
  // cross-attention maps (parseq_forward_args.attn_maps): the query stream of the last layer writes the head-averaged
  // weights of row (b, qi) to maps + (b * nq + qi) * T.  With cand_off the maps have maps_ld rows per candidate, rows
  // past maps_len[c] (the group's candidate lengths, device) written as 0 (dec_cross_attn_maps_grouped_kernel)
  float* maps = nullptr;
  const int* maps_len = nullptr;
  int maps_ld = 0;
  Tail tail = Tail::Head;
  // Head: row r's logits at logits + r * logits_ld; with ids_dst the greedy id of row (b, qi) goes to
  // ids_dst[b * ids_ld + dst_off + qi], or with `forced` (teacher forcing) forced[b * forced_ld + dst_off + qi].
  // Head and TopK: `mask` holds the images' class allowlist rows, or null
  float* logits = nullptr;
  long long logits_ld = 0;
  const uint32_t* mask = nullptr;
  int* ids_dst = nullptr;
  const int* forced = nullptr;
  int dst_off = 0, forced_ld = 0;
  const int* lse_tgt = nullptr;          // LogSumExp: [B*nq] target class per row
  float2* part = nullptr;                // TopK: k keys per row and 128-class tile, the allowlist row of r is image r / beam
  unsigned long long* keys = nullptr;
  int k = 0;
  float* out_norm = nullptr;             // Norm: [B*nq, D] fp32
};

// A stream's self-attention mask: Caller where the pass has a padding mask or the stream's own mask (content stream:
// cmask, query stream: qmask), or in the query stream the caller's queries; else the pass's own
SelfMask self_mask(const DecodePass& p, bool content) {
  const bool caller = p.pmask != nullptr || (content ? p.cmask != nullptr : p.qmask != nullptr || p.query != nullptr);
  return caller ? SelfMask::Caller : p.self_mask;
}

const __nv_bfloat16* ckv_of(const parseq_engine* e, int layer) { return layer == 0 ? e->ckv : e->ckv_deep[layer - 1]; }

// Calls f(std::integral_constant<int, TB>) with the 128-token blocks of the image memory that the decoder's
// cross-attention kernels are instantiated for: TB = 1 up to 128 tokens, else 2 (NR = 4 TB keys per lane)
template <typename F>
int dispatch_tokens(int T, F&& f) {
  return T <= 128 ? f(std::integral_constant<int, 1>{}) : f(std::integral_constant<int, 2>{});
}

// Self-attention sg.qc -> sg.sa of layer l with one query row per (image, query) (decoders of depth >= 2), nq rows per
// image from position q0 of the content or query stream, over the (position, token) table (l = 0) or the layer's cache.
int self_attn_rows(parseq_engine* e, parseq_engine::Stage& sg, const DecodePass& p, int l, bool content, int nq, int q0,
                   cudaStream_t st) {
  const int D = e->D;
  TimedScope ts(e, st, CAT_DEC_ATTN, 4.0 * p.B * nq * p.nkeys * D);
  const int qsplit = (nq >= 8) ? 4 : 1;
  const bool cache = l > 0;
  auto kern = e->ids_ld == 32 ? (cache ? pq::dec_self_attn2_rows_kernel<true> : pq::dec_self_attn2_rows_kernel<false>)
                              : (cache ? pq::dec_self_attn2_rows_long_kernel<true> : pq::dec_self_attn2_rows_long_kernel<false>);
  const __nv_bfloat16* kv = cache ? sg.kvc[l - 1] : e->kvtab;
  return launch_k(e->lo, kern, dim3(p.B * qsplit), dim3(D < 384 ? D : 384), 0, st, static_cast<const float*>(sg.qc), kv, p.ids,
                  e->ids_ld, cache ? p.kv_pitch(e) : e->V, D, nq, q0, p.nkeys, static_cast<int>(self_mask(p, content)),
                  /*eos*/ 0, sg.sa, qsplit, content ? p.cmask : p.qmask, p.pmask);
}

// The rest of decoder layer `l` after its self-attention (modules.py:72-78) on a residual stream x [p.B * nq, D] (fp32, in
// place): x += out_proj(sa); x += cross_attn(norm1(x)); x += MLP(norm2(x)).  add != null: x holds no residual yet, the
// base is the broadcast table / caller rows `add` (row r adds add[r % add_mod]).  With `maps_layer` the layer writes the
// pass's maps (a MapsOnly pass ends there).
int dec_layer_rest(parseq_engine* e, parseq_engine::Stage& sg, const DecodePass& p, int l, int nq, float* x, const float* add,
                   int add_mod, bool maps_layer, cudaStream_t st) {
  const int D = e->D, M = p.B * nq;
  const int B = p.B / p.beam;             // images; each has p.beam * nq query rows
  nq *= p.beam;
  const std::string Ly = "decoder.layers." + std::to_string(l) + ".";
  const float qscale = 1.0f / std::sqrt(static_cast<float>(e->dh_dec));
  if (add != nullptr) {
    // y = query + out_proj(sa): the GEMM stores out_proj(sa) with its TMA epilogue, the LayerNorm kernel adds the query
    // residual (broadcast pos_queries[q0 + qi], or the caller's rows), writes y back and emits norm1(y)
    PQ_TRY(gemm(e, sg.sa, D, e->w(Ly + "self_attn.out_proj.weight"), D, e->wf(Ly + "self_attn.out_proj.bias"), M, D, D,
                pq::EPI_F32, 1.0f, nullptr, 0, 0, x, D, st));
    PQ_TRY(layernorm(e, x, Ly + "norm1", 1e-5f, M, sg.yn, nullptr, st, add, add_mod, x));
  } else {
    PQ_TRY(gemm(e, sg.sa, D, e->w(Ly + "self_attn.out_proj.weight"), D, e->wf(Ly + "self_attn.out_proj.bias"), M, D, D,
                pq::EPI_F32, 1.0f, x, D, 0, x, D, st));
    PQ_TRY(layernorm(e, x, Ly + "norm1", 1e-5f, M, sg.yn, nullptr, st));
  }
  PQ_TRY(gemm(e, sg.yn, D, e->wb(Ly + "cross_attn.in_proj_weight"), D, e->wf(Ly + "cross_attn.in_proj_bias"), M, D, D,
              pq::EPI_F32, qscale, nullptr, 0, 0, sg.qc, D, st));
  const long long kv_rows = 1ll * e->max_batch * e->T;
  const int H = e->cfg.dec_num_heads;
  const float* q = sg.qc;
  if (maps_layer && p.maps != nullptr) {
    // the head-averaged weights of these query rows, from the q just projected and the layer's K (reads only)
    TimedScope ts(e, st, CAT_MAPS, 2.0 * M * e->T * D);
    PQ_TRY(dispatch_tokens(e->T, [&](auto tb) {
      constexpr int NR = 4 * decltype(tb)::value;
      if (p.cand_off != nullptr) {
        // candidate scoring: every image's candidates' maps_ld map rows, at most cand_max_rows / nq candidates per image
        const int max_rows = p.cand_max_rows / nq * p.maps_ld;
        const dim3 grid(static_cast<unsigned>(p.cand_imgs), static_cast<unsigned>((max_rows + pq::AMAP_ROWS - 1) / pq::AMAP_ROWS));
        return launch_k(e->lo, pq::dec_cross_attn_maps_grouped_kernel<NR>, grid, dim3(pq::AMAP_THREADS), 0, st, q, ckv_of(e, l),
                        kv_rows, p.b_first, e->T, D, H, nq, p.cand_off, p.maps_len, p.maps_ld, p.maps);
      }
      const dim3 grid(static_cast<unsigned>(B), static_cast<unsigned>((nq + pq::AMAP_ROWS - 1) / pq::AMAP_ROWS));
      return launch_k(e->lo, pq::dec_cross_attn_maps_kernel<NR>, grid, dim3(pq::AMAP_THREADS), 0, st, q, ckv_of(e, l), kv_rows,
                      p.b_first, e->T, D, H, nq, p.maps);
    }));
    if (p.tail == Tail::MapsOnly) return PARSEQ_OK;
  }
  {
    TimedScope ts(e, st, CAT_DEC_ATTN, 4.0 * M * e->T * D);
    PQ_TRY(dispatch_tokens(e->T, [&](auto tb) {
      constexpr int NR = 4 * decltype(tb)::value;
      if (p.cand_off != nullptr) {
        // candidate scoring: the rows of each image's candidates attend to that image (64 rows per CTA)
        constexpr int kRows = 64;
        const dim3 grid(static_cast<unsigned>(p.cand_imgs * H), static_cast<unsigned>((p.cand_max_rows + kRows - 1) / kRows));
        return launch_k(e->lo, pq::dec_cross_attn3_grouped_kernel<NR>, grid, dim3(128), 0, st, q, ckv_of(e, l), kv_rows,
                        p.b_first, e->T, D, H, nq, p.cand_off, kRows, sg.ca);
      }
      return launch_k(e->lo, pq::dec_cross_attn3_kernel<NR>, dim3(B * H), dim3(128), 0, st, q, ckv_of(e, l), kv_rows, p.b_first,
                      e->T, D, H, nq, sg.ca);
    }));
  }
  PQ_TRY(gemm(e, sg.ca, D, e->w(Ly + "cross_attn.out_proj.weight"), D, e->wf(Ly + "cross_attn.out_proj.bias"), M, D, D,
              pq::EPI_F32, 1.0f, x, D, 0, x, D, st));
  PQ_TRY(layernorm(e, x, Ly + "norm2", 1e-5f, M, sg.yn, nullptr, st));
  PQ_TRY(gemm(e, sg.yn, D, e->w(Ly + "linear1.weight"), D, e->wf(Ly + "linear1.bias"), M, e->Md, D, pq::EPI_GELU_BF16,
              1.0f, nullptr, 0, 0, sg.hd, e->Md, st));
  PQ_TRY(gemm(e, sg.hd, e->Md, e->w(Ly + "linear2.weight"), e->Md, e->wf(Ly + "linear2.bias"), M, D, e->Md, pq::EPI_F32,
              1.0f, x, D, 0, x, D, st));
  return PARSEQ_OK;
}

// Content stream of a decoder of depth >= 2 (modules.py:94-97, 119-123): context rows [k0, k0 + nc) of the pass's B
// rows through layers 0..depth-2, each appending its K/V rows of the next layer to that layer's cache (row b * pitch + k).
// An AR step computes its own position's row (nc = 1, pitch L: the causal content rows of earlier positions do not change
// as the context grows), any other pass its whole context (nc = nkeys = pitch).  The content rows attend to keys
// 0..nkeys-1 under the pass's mask, or under the caller's content / padding masks (self_mask).  Beam rows (nc = 1) are
// p.beam consecutive rows per image.
int content_stream(parseq_engine* e, parseq_engine::Stage& sg, const DecodePass& p, cudaStream_t st) {
  const int k0 = p.ar_step ? p.q0 : 0, nc = p.ar_step ? 1 : p.nkeys, pitch = p.kv_pitch(e);
  const int D = e->D, M = p.B * nc;
  const float qscale = 1.0f / std::sqrt(static_cast<float>(e->dh_dec));
  {
    TimedScope ts(e, st, CAT_MISC, 0.0);
    const long long total = 1ll * M * D;
    PQ_TRY(launch_k(e->lo, pq::gather_ctx_rows_kernel, dim3(static_cast<unsigned>(std::min<long long>((total + 255) / 256, 132ll * 8))),
                    dim3(256), 0, st, e->wf("text_embed.embedding.weight"), e->wf("pos_queries"), p.ids, e->ids_ld, p.B, k0, nc, D,
                    std::sqrt(static_cast<float>(D)), sg.cx));
  }
  PQ_TRY(layernorm(e, sg.cx, "decoder.layers.0.norm_c", 1e-5f, M, sg.yn, nullptr, st));
  const long long ldo = (nc == pitch ? 1ll : pitch) * 2 * D;
  for (int l = 0; l + 1 < e->cfg.dec_depth; ++l) {
    // sg.yn = norm_c_l(content_l): the content queries of layer l (its keys are the same rows' K/V, already stored)
    const std::string Ly = "decoder.layers." + std::to_string(l) + ".";
    PQ_TRY(gemm(e, sg.yn, D, e->w(Ly + "self_attn.in_proj_weight"), D, e->wf(Ly + "self_attn.in_proj_bias"), M, D, D,
                pq::EPI_F32, qscale, nullptr, 0, 0, sg.qc, D, st));
    PQ_TRY(self_attn_rows(e, sg, p, l, /*content*/ true, nc, k0, st));
    PQ_TRY(dec_layer_rest(e, sg, p, l, nc, sg.cx, nullptr, 0, /*maps_layer*/ false, st));
    // K/V of layer l + 1 = W_kv norm_c_{l+1}(content_{l+1}) + b_kv, into rows k0.. of its cache
    const std::string Ln = "decoder.layers." + std::to_string(l + 1) + ".";
    PQ_TRY(layernorm(e, sg.cx, Ln + "norm_c", 1e-5f, M, sg.yn, nullptr, st));
    PQ_TRY(gemm(e, sg.yn, D, e->wb(Ln + "self_attn.in_proj_weight") + 1ll * D * D, D, e->wf(Ln + "self_attn.in_proj_bias") + D,
                M, 2 * D, D, pq::EPI_BF16, 1.0f, nullptr, 0, 0, sg.kvc[l] + 2ll * k0 * D, ldo, st));
  }
  return PARSEQ_OK;
}

// The decoder on the pass's rows: the content stream (depth >= 2), the query stream of every layer, then the tail.
int decode_pass(parseq_engine* e, parseq_engine::Stage& sg, const DecodePass& p, cudaStream_t st) {
  if (p.tail == Tail::MapsOnly && p.maps == nullptr) return fail(PARSEQ_ERR_STATE, "decode_pass: a maps-only pass needs maps");
  const int D = e->D, B = p.B, nq = p.nq, M = B * nq;
  const std::string Ly = "decoder.layers.0.";
  const float qscale = 1.0f / std::sqrt(static_cast<float>(e->dh_dec));
  e->cur_cat = CAT_DEC_GEMM;
  if (e->cfg.dec_depth > 1) PQ_TRY(content_stream(e, sg, p, st));
  const float* qself = e->qs;            // [L, D] table of W_q LN_q(pos_queries), pre-scaled
  const SelfMask mode = self_mask(p, /*content*/ false);
  if (p.query != nullptr) {
    // custom queries: q = scale * (W_q LN_q(query) + b_q), one row per (image, query)
    PQ_TRY(layernorm(e, p.query, Ly + "norm_q", 1e-5f, M, sg.yn, nullptr, st));
    PQ_TRY(gemm(e, sg.yn, D, e->w(Ly + "self_attn.in_proj_weight"), D, e->wf(Ly + "self_attn.in_proj_bias"), M, D, D,
                pq::EPI_F32, qscale, nullptr, 0, 0, sg.qc, D, st));
    qself = sg.qc;
  } else if (mode == SelfMask::Caller) {
    // masks with the default queries: expand the table rows (tiny) so that mode 2 finds one query row per (image, query).
    // Launched without PDL: the kernel has no griddepcontrol.wait, so as a PDL launch it could start under the previous
    // kernel on the stream (an early-triggering GEMM: the cross K/V, or the previous scoring group's head), and every
    // later kernel of this pass, which waits only for its own predecessor, would lose its order after that kernel
    const int n4 = nq * D / 4;
    PQ_TRY(launch_ex(LaunchConfig(dim3(static_cast<unsigned>(std::min((B * n4 + 255) / 256, 132 * 8))), dim3(256), 0, st, 0, false),
                     pq::bcast_rows_kernel, reinterpret_cast<const float4*>(e->qs + static_cast<long long>(p.q0) * D),
                     reinterpret_cast<float4*>(sg.qc.get()), n4, B));
    e->launches++;
    qself = sg.qc;
  }
  {
    TimedScope ts(e, st, CAT_DEC_ATTN, 4.0 * M * p.nkeys * D);
    const int qsplit = (nq >= 8) ? 4 : 1;
    // one key per lane up to 32 keys, two up to 64 (the kernel of the engine's id pitch)
    PQ_TRY(launch_k(e->lo, e->ids_ld == 32 ? pq::dec_self_attn2_kernel : pq::dec_self_attn2_long_kernel, dim3(B * qsplit),
                    dim3(D < 384 ? D : 384), 0, st, qself, static_cast<const __nv_bfloat16*>(e->kvtab), p.ids, e->ids_ld, e->V,
                    D, nq, p.q0, p.nkeys, static_cast<int>(mode), /*eos*/ 0, sg.sa, qsplit, p.qmask, p.pmask));
  }
  const float* resid = p.query != nullptr ? p.query : e->wf("pos_queries") + static_cast<long long>(p.q0) * D;
  const int last = e->cfg.dec_depth - 1;
  PQ_TRY(dec_layer_rest(e, sg, p, 0, nq, sg.y, resid, p.query != nullptr ? M : nq, last == 0, st));
  // query stream of layers >= 1 (modules.py:91-93): its residual base is the previous layer's output, its keys the
  // layer's content K/V cache
  for (int l = 1; l < e->cfg.dec_depth; ++l) {
    const std::string Ll = "decoder.layers." + std::to_string(l) + ".";
    PQ_TRY(layernorm(e, sg.y, Ll + "norm_q", 1e-5f, M, sg.yn, nullptr, st));
    PQ_TRY(gemm(e, sg.yn, D, e->w(Ll + "self_attn.in_proj_weight"), D, e->wf(Ll + "self_attn.in_proj_bias"), M, D, D,
                pq::EPI_F32, qscale, nullptr, 0, 0, sg.qc, D, st));
    PQ_TRY(self_attn_rows(e, sg, p, l, /*content*/ false, nq, p.q0, st));
    PQ_TRY(dec_layer_rest(e, sg, p, l, nq, sg.y, nullptr, 0, l == last, st));
  }
  if (p.tail == Tail::MapsOnly) return PARSEQ_OK;   // dec_layer_rest stopped after the last layer's maps
  if (p.tail == Tail::Head && nq == 1 && e->C <= 128) {
    TimedScope ts(e, st, CAT_DEC_GEMM, 2.0 * M * e->C * D);
    return ln_head_argmax_launch(e->lo, sg.y, e->wf("decoder.norm.weight"), e->wf("decoder.norm.bias"), 1e-5f,
                                 e->wb("head.weight"), e->wf("head.bias"), M, e->C, D, p.logits, p.logits_ld, p.ids_dst,
                                 e->ids_ld, nq, p.dst_off, p.forced, p.forced_ld, p.mask, st);
  }
  // decoder.norm (modules.py:123-125): PARSeq.decode returns it (Norm), every other tail feeds it to the head
  PQ_TRY(layernorm(e, sg.y, "decoder.norm", 1e-5f, M, sg.yn, p.tail == Tail::Norm ? p.out_norm : nullptr, st));
  if (p.tail == Tail::Norm) return PARSEQ_OK;
  if (p.tail == Tail::LogSumExp) {
    // candidate scoring: the head GEMM's epilogue keeps only the per-row log-sum-exp partials and target logits
    // (score_reduce_kernel finishes the terms)
    TimedScope ts(e, st, CAT_SCORE, 2.0 * M * e->C * D);
    return gemm_lse_launch(e->lo, sg.yn, D, e->w("head.weight"), D, e->wf("head.bias"), M, e->C, D, p.lse_tgt, sg.lse_part,
                           sg.lse_tlogit, st);
  }
  if (p.tail == Tail::TopK) {
    TimedScope ts(e, st, CAT_DEC_GEMM, 2.0 * M * e->C * D);
    return gemm_topk_launch(e->lo, sg.yn, D, e->w("head.weight"), D, e->wf("head.bias"), M, e->C, D, p.k, p.mask, p.beam,
                            p.part, p.keys, st);
  }
  // Head of a multi-query pass (refine / NAR) or too large for the fused kernel's shared memory: the wgmma GEMM (weights
  // read once per tile), then the greedy argmax if ids are asked for.  Chosen by pass type, not by batch size, so that a
  // row's result does not depend on the batch it is computed in.
  PQ_TRY(gemm(e, sg.yn, D, e->w("head.weight"), D, e->wf("head.bias"), M, e->C, D, pq::EPI_F32, 1.0f, nullptr, 0, 0, p.logits,
              p.logits_ld, st));
  if (p.ids_dst != nullptr)
    PQ_TRY(argmax_rows(e, p.logits, static_cast<int>(p.logits_ld / e->C), B, nq, 0, p.ids_dst, e->ids_ld, p.dst_off, p.forced,
                       p.forced_ld, p.mask, st));
  return PARSEQ_OK;
}

// Greedy ids of B images x nrows logits rows; with an allowlist (`mask`: the images' rows) the disallowed logits are set to
// -inf in place first, and `ids` may be null.
int argmax_rows(parseq_engine* e, float* logits, int L, int B, int nrows, int src0, int* ids, int ids_ld, int dst0,
                const int* forced, int forced_ld, const uint32_t* mask, cudaStream_t st) {
  const int warps = B * nrows;
  if (warps <= 0) return PARSEQ_OK;
  TimedScope ts(e, st, CAT_MISC, 0.0);
  return launch_k(e->lo, pq::argmax_rows_kernel, dim3((warps + 7) / 8), dim3(256), 0, st, logits, L, e->C, B, nrows, src0, ids, ids_ld,
                  dst0, forced, forced_ld, mask);
}

// The cross-attention maps of an AR-only schedule (no refinement): row i is AR step i's query.  Under teacher forcing
// step i is a fixed function of the memory and the context 0..i, so one pass over the AR loop's own ids
// [BOS, ids[:, :L-1]] (`ids`: its [B, ids_ld] id rows) under the causal query mask, and at depth >= 2 the causal content
// mask, computes every step's query at once (the argument parseq_score rests on).  It stops after the last layer's maps
// and writes nothing else the caller sees; whichever AR loop ran, the maps depend only on the ids.  beam > 1 (beam
// search): the B rows are `beam` consecutive hypotheses of each image.
int ar_maps_pass(parseq_engine* e, parseq_engine::Stage& sg, int b_first, int B, int L, const int* ids, float* maps,
                 cudaStream_t st, int beam = 1) {
  const unsigned char* causal = e->sc_causal + 1ll * (L - 1) * e->L * e->L;
  DecodePass p;
  p.b_first = b_first; p.B = B; p.nq = L; p.nkeys = L; p.ids = ids; p.beam = beam;
  p.qmask = causal; p.cmask = e->cfg.dec_depth > 1 ? causal : nullptr;
  p.maps = maps; p.tail = Tail::MapsOnly;
  return decode_pass(e, sg, p, st);
}

// id rows [B, ids_ld] = BOS, PAD, PAD, ...: the context of a first AR step or of a NAR / refinement pass
int fill_ids(parseq_engine* e, int* ids, int B, cudaStream_t st) {
  PQ_TRY(launch_k(e->lo, pq::fill_ids_kernel, dim3((B * e->ids_ld + 255) / 256), dim3(256), 0, st, ids, B, e->ids_ld, e->V - 2,
                  e->V - 1));
  e->launches++;
  return PARSEQ_OK;
}

// Decoder chain of one group of B <= dec_chunk images (their cross K/V is at `ckv`): AR loop / NAR pass, cloze
// refinement, final argmax.  model.py:113-169.  `mask`: the group's class allowlist rows, or null.  Every head output
// that the multi-query passes (and the chain's large-head AR steps) leave unmasked is masked by the argmax that reads it,
// and the final argmax runs with a mask even when the caller wants no ids, so no unmasked logit is returned.
// `maps` (the group's [B, L, T] cross-attention maps, or null): written by the pass that produced the returned logits.
int decode_stage(parseq_engine* e, parseq_engine::Stage& sg, int b_first, const parseq_forward_args* a, int b0,
                 int B, int L, float* logits, int* ids_out, int* steps, const uint32_t* mask, cudaStream_t st, bool ar_done,
                 float* maps) {
  // b_first: index of the group's first image inside the super-chunk (row of the K/V cache); b0: inside the caller's batch
  const int C = e->C;
  const bool testing = a->max_length < 0;
  DecodePass chain;                 // what the chain's passes share: their rows, Head tails into [B, L, C] logits
  chain.b_first = b_first; chain.B = B; chain.logits = logits; chain.logits_ld = C; chain.mask = mask;
  if (a->decode_ar && ar_done) {
    // the AR loop of the whole super-chunk already ran in the persistent kernel (ar_decode)
  } else if (a->decode_ar) {
    PQ_TRY(fill_ids(e, sg.ids_ar, B, st));
    DecodePass p = chain;
    p.nq = 1; p.ids = sg.ids_ar; p.ar_step = true;
    p.logits_ld = static_cast<long long>(L) * C;
    p.forced = a->forced_ids ? a->forced_ids + static_cast<long long>(b0) * L : nullptr; p.forced_ld = L;
    for (int i = 0; i < L; ++i) {
      // step i: context ids[:, :i+1], query position i; the head writes ids[:, i+1] = argmax (model.py:142)
      p.q0 = i; p.nkeys = i + 1;
      p.logits = logits + static_cast<long long>(i) * C;
      p.ids_dst = i + 1 < L ? sg.ids_ar.get() : nullptr; p.dst_off = i + 1;
      PQ_TRY(decode_pass(e, sg, p, st));
    }
    if (testing && steps != nullptr) {
      PQ_TRY(launch_k(e->lo, pq::ar_steps_kernel, dim3(1), dim3(256), 0, st, static_cast<const int*>(sg.ids_ar), e->ids_ld, B, L,
                      0, steps));
      e->launches++;
    }
  } else {
    PQ_TRY(fill_ids(e, sg.ids_ctx, B, st));
    DecodePass p = chain;
    p.nq = L; p.nkeys = 1; p.ids = sg.ids_ctx;
    p.maps = a->refine_iters == 0 ? maps : nullptr;
    PQ_TRY(decode_pass(e, sg, p, st));
  }
  for (int it = 0; it < a->refine_iters; ++it) {
    PQ_TRY(fill_ids(e, sg.ids_ctx, B, st));
    const int* forced = a->forced_refine
                            ? a->forced_refine + (static_cast<long long>(it) * a->batch + b0) * L
                            : nullptr;
    // ctx = [BOS, argmax(logits[:, :L-1])]  (model.py:161)
    PQ_TRY(argmax_rows(e, logits, L, B, L - 1, 0, sg.ids_ctx, e->ids_ld, 1, forced, L, mask, st));
    DecodePass p = chain;
    p.nq = L; p.nkeys = L; p.ids = sg.ids_ctx; p.self_mask = SelfMask::Cloze;
    p.maps = it + 1 == a->refine_iters ? maps : nullptr;
    PQ_TRY(decode_pass(e, sg, p, st));
  }
  if (ids_out != nullptr || mask != nullptr) PQ_TRY(argmax_rows(e, logits, L, B, L, 0, ids_out, L, 0, nullptr, 0, mask, st));
  if (maps != nullptr && a->decode_ar && a->refine_iters == 0) PQ_TRY(ar_maps_pass(e, sg, b_first, B, L, sg.ids_ar, maps, st));
  return PARSEQ_OK;
}


// ---- which implementation runs the AR loop ----
// Why the grid-barrier kernel (dec_ar.cuh) cannot take this engine's AR loop, or nullptr if it can.
const char* grid_barrier_limit(const parseq_engine* e) {
  if (e->C > 128) return "ar_kernel = 1 (grid-barrier AR kernel) covers at most 128 head classes; use ar_kernel 0 or 2";
  if (e->L > 32) return "ar_kernel = 1 (grid-barrier AR kernel) covers max_label_length <= 31; use ar_kernel 0 or 2";
  if (e->cfg.dec_depth > 1) return "ar_kernel = 1 (grid-barrier AR kernel) covers dec_depth 1; use ar_kernel 0 or 2";
  return nullptr;
}
enum class ArPath { Chain, GridBarrier, Cluster };
// Option "ar_kernel" 2 (default) runs the cluster kernel (dec_ar2.cuh) where it applies: heads of <= 96 classes run
// redundantly in every CTA, > 128 classes take the class-sliced head.  Anything else it cannot take (97..128 classes,
// dec_mlp_ratio != 4) runs on the grid-barrier kernel if that holds it, else on the chain of separate kernels, as do
// decoders of depth >= 2.  "ar_kernel" 1 (accepted only where the grid-barrier kernel applies) forces that kernel, 0 the
// chain.
ArPath ar_path(const parseq_engine* e) {
  if (e->arch != 0 || e->ar_kernel == 0) return ArPath::Chain;
  if (e->ar_kernel == 2 && e->cfg.dec_depth == 1 && e->cfg.dec_mlp_ratio == 4 && (e->C <= 96 || e->C > 128) && e->T <= 256 &&
      e->dh_dec == 32)
    return ArPath::Cluster;
  if (grid_barrier_limit(e) == nullptr) return ArPath::GridBarrier;
  return ArPath::Chain;
}

// ---- cluster-owned AR kernel (dec_ar2.cuh) ----
bool ar2_wide(const parseq_engine* e) { return e->C > 128; }
// weight descriptors: once per weight set (parseq_finalize); K/V cache descriptor: once per workspace
int ar2_build_maps(parseq_engine* e) {
  const int D = e->D;
  const std::string Ly = "decoder.layers.0.";
  for (int ci = 0; ci < 2; ++ci) {
    const int cs = ci == 0 ? 8 : 6;
    pq::DecAr2Maps& m = e->ar2_maps[ci];
    const int DS = D / cs, MS = e->Md / cs;
    const int NC1 = (MS % 128 == 0) ? 128 : 96, NC2 = (D % 128 == 0) ? 128 : 96;
    PQ_TRY(make_tmap(&m.wo_s, e->w(Ly + "self_attn.out_proj.weight"), 2, D, D, D, 64, DS));
    PQ_TRY(make_tmap(&m.wq_c, e->w(Ly + "cross_attn.in_proj_weight"), 2, D, D, D, 64, DS));
    PQ_TRY(make_tmap(&m.wo_c, e->w(Ly + "cross_attn.out_proj.weight"), 2, D, D, D, 64, DS));
    PQ_TRY(make_tmap(&m.w1, e->w(Ly + "linear1.weight"), 2, e->Md, D, D, 64, NC1));
    PQ_TRY(make_tmap(&m.w2, e->w(Ly + "linear2.weight"), 2, D, e->Md, e->Md, 64, NC2));
    PQ_TRY(make_tmap(&m.wh, e->w("head.weight"), 2, e->C, D, D, 64, ar2_wide(e) ? 128 : 96));
    const int tbox = e->T <= 64 ? 64 : 128;
    PQ_TRY(make_tmap_kv4d(&m.ckv, e->ckv, e->T, e->max_batch, 2 * D / 64, tbox));
  }
  e->ar2_maps_ok = true;
  return PARSEQ_OK;
}
// ncl clusters of CS CTAs; the AR kernel is never launched with PDL
template <int D, int MT, int CS, int IDP>
LaunchConfig ar2_config(int ncl, cudaStream_t st) {
  return LaunchConfig(dim3(static_cast<unsigned>(ncl * CS)), dim3(pq::A2_LAUNCH_THREADS), pq::dec_ar2_smem_bytes<D, MT, CS, IDP>(),
                      st, CS, false);
}
template <int D, int MT, int CS, bool WIDE, int IDP>
int ar2_launch_t(parseq_engine* e, const pq::DecAr2Params& p, int ncl, cudaStream_t st) {
  const LaunchConfig lc = ar2_config<D, MT, CS, IDP>(ncl, st);
  e->ar_last_per = p.per; e->ar_last_ncl = ncl; e->ar_last_cs = CS;
  e->ar_last_mt = MT; e->ar_last_hs = 0; e->ar_last_wide = WIDE ? 1 : 0; e->ar_last_idp = IDP;
  if constexpr (MT == 1 && CS == 8 && D / 64 <= CS) {
    // so few images per cluster that (images x head pairs) fit its CTAs: every CTA takes one (image, head pair) of the
    // cross-attention instead of whole images (bs = 1: 9 -> 2.5 us per step; same bits per head)
    if (p.per * (D / 64) <= CS) {
      e->ar_last_hs = 1;
      return launch_ex(lc, ar2_kernel<D, MT, CS, true, WIDE, IDP>(), e->ar2_maps[0], p);
    }
  }
  return launch_ex(lc, ar2_kernel<D, MT, CS, false, WIDE, IDP>(), e->ar2_maps[CS == 6 ? 1 : 0], p);
}
template <int D, int MT, int CS, int IDP>
int ar2_launch(parseq_engine* e, const pq::DecAr2Params& p, int ncl, cudaStream_t st) {
  return ar2_wide(e) ? ar2_launch_t<D, MT, CS, true, IDP>(e, p, ncl, st) : ar2_launch_t<D, MT, CS, false, IDP>(e, p, ncl, st);
}
// Clusters of this instantiation that can be co-resident, as the occupancy query answers for this device.  A cluster
// lives inside one GPC, so clusters of 8 can leave SMs of a GPC idle and clusters of 6 may pack more SMs; a batch that
// needs more clusters than fit runs in two waves.
template <int D, int MT, int CS, int IDP>
int ar2_max_clusters(parseq_engine* e) {
  int& cache = e->ar2_clusters[MT][CS == 6 ? 1 : 0];
  if (cache > 0) return cache;
  const LaunchConfig lc = ar2_config<D, MT, CS, IDP>(e->lo.sm_count / CS, nullptr);
  int n = 0;
  // (the cache is per engine, and so are the head width and the id pitch)
  const cudaError_t qe = ar2_wide(e) ? cudaOccupancyMaxActiveClusters(&n, ar2_kernel<D, MT, CS, false, true, IDP>(), &lc.cfg)
                                     : cudaOccupancyMaxActiveClusters(&n, ar2_kernel<D, MT, CS, false, false, IDP>(), &lc.cfg);
  if (qe != cudaSuccess || n <= 0) {
    cudaGetLastError();
    n = (CS == 8) ? (e->lo.sm_count / 10) : 1;   // unknown: a conservative guess for 8, "do not use" for 6
  }
  e->ar2_occ[MT][CS == 6 ? 1 : 0] = n;
  if (e->ar_clusters_override > 0) n = e->ar_clusters_override;
  cache = n;
  return n;
}
// Spread the batch over the co-resident clusters.  Candidates in order of per-step cost: clusters of 8 with one m16 row
// tile, clusters of 8 with two, clusters of 6 (a third more weight bytes per CTA and step); the first that holds the
// batch in ONE wave wins (the loop is latency-bound: a second wave doubles its time), else the fewest waves.
template <int D, int IDP>
int ar2_dispatch(parseq_engine* e, pq::DecAr2Params& p, cudaStream_t st) {
  constexpr bool kHas2 = (D != 768);            // two m16 tiles of D = 768 rows do not fit shared memory
  struct Cand { int mt, cs, maxc, rows; };
  Cand c[4];
  int nc = 0;
  const bool allow6 = e->ar_cs != 8, allow8 = e->ar_cs != 6;
  if (allow8) c[nc++] = Cand{1, 8, ar2_max_clusters<D, 1, 8, IDP>(e), 16};
  if constexpr (kHas2) { if (allow8) c[nc++] = Cand{2, 8, ar2_max_clusters<D, 2, 8, IDP>(e), 32}; }
  if (allow6) c[nc++] = Cand{1, 6, ar2_max_clusters<D, 1, 6, IDP>(e), 16};
  if constexpr (kHas2) { if (allow6) c[nc++] = Cand{2, 6, ar2_max_clusters<D, 2, 6, IDP>(e), 32}; }
  int best = -1, best_waves = 1 << 30;
  for (int i = 0; i < nc; ++i) {
    const int need = (p.B + c[i].rows - 1) / c[i].rows;             // clusters at full rows
    const int waves = (need + c[i].maxc - 1) / c[i].maxc;
    if (waves < best_waves) { best = i; best_waves = waves; }
  }
  const Cand& k = c[best];
  int per = (p.B + k.maxc * best_waves - 1) / (k.maxc * best_waves);   // even spread over the clusters of all waves
  if (per > k.rows) per = k.rows;
  if (per < 1) per = 1;
  p.per = per;
  const int ncl = (p.B + per - 1) / per;
  if (k.cs == 8) {
    if (k.mt == 1) return ar2_launch<D, 1, 8, IDP>(e, p, ncl, st);
    if constexpr (kHas2) return ar2_launch<D, 2, 8, IDP>(e, p, ncl, st);
  } else {
    if (k.mt == 1) return ar2_launch<D, 1, 6, IDP>(e, p, ncl, st);
    if constexpr (kHas2) return ar2_launch<D, 2, 6, IDP>(e, p, ncl, st);
  }
  return fail(PARSEQ_ERR_STATE, "dec_ar2: no launch configuration");
}

// The whole AR loop (model.py:119-147) of B images in one persistent launch: the cluster kernel (dec_ar2.cuh) or the
// grid-barrier kernel (dec_ar.cuh), as ar_path chose.
int ar_decode(parseq_engine* e, ArPath path, const parseq_forward_args* a, int b0, int B, int L, float* logits, int* steps,
              const uint32_t* mask, cudaStream_t st) {
  const int D = e->D;
  const std::string Ly = "decoder.layers.0.";
  PQ_TRY(fill_ids(e, e->ar_ids, B, st));
  // what both kernels read: the decoder's tables, bias and LayerNorm vectors, the id rows and the logits
  auto common = [&](auto& p) {
    p.B = B; p.L = L; p.V = e->V; p.C = e->C; p.T = e->T;
    p.qscale = 1.0f / std::sqrt(static_cast<float>(e->dh_dec));
    p.qs = e->qs; p.kvtab = e->kvtab; p.posq = e->wf("pos_queries");
    p.bo_s = e->wf(Ly + "self_attn.out_proj.bias"); p.bq_c = e->wf(Ly + "cross_attn.in_proj_bias");
    p.bo_c = e->wf(Ly + "cross_attn.out_proj.bias"); p.b1 = e->wf(Ly + "linear1.bias"); p.b2 = e->wf(Ly + "linear2.bias");
    p.bh = e->wf("head.bias");
    p.g1 = e->wf(Ly + "norm1.weight"); p.be1 = e->wf(Ly + "norm1.bias");
    p.g2 = e->wf(Ly + "norm2.weight"); p.be2 = e->wf(Ly + "norm2.bias");
    p.g3 = e->wf("decoder.norm.weight"); p.be3 = e->wf("decoder.norm.bias");
    p.ids = e->ar_ids; p.ids_ld = e->ids_ld; p.logits = logits;
    p.forced = a->forced_ids ? a->forced_ids + static_cast<long long>(b0) * L : nullptr;
    p.forced_ld = L;
    p.mask = mask;
    p.prof = e->ar_prof_on ? e->ar_prof.get() : nullptr;
  };
  pq::DecAr2Params q;
  pq::DecArParams p;
  if (path == ArPath::Cluster) {
    if (!e->ar2_maps_ok) PQ_TRY(ar2_build_maps(e));
    common(q);
    q.per = 0;
    q.tbox = e->T <= 64 ? 64 : 128; q.tb = (e->T + 127) / 128;
  } else {
    PQ_CUDA(cudaMemsetAsync(e->ar_bar, 0, 64, st));
    common(p);
    p.Md = e->Md; p.heads = e->cfg.dec_num_heads;
    p.Wo_s = e->wb(Ly + "self_attn.out_proj.weight"); p.Wq_c = e->wb(Ly + "cross_attn.in_proj_weight");
    p.Wo_c = e->wb(Ly + "cross_attn.out_proj.weight"); p.W1 = e->wb(Ly + "linear1.weight"); p.W2 = e->wb(Ly + "linear2.weight");
    p.Wh = e->wb("head.weight");
    p.ckv = e->ckv; p.kv_rows = 1ll * e->max_batch * e->T;
    p.sa = e->ar_sa; p.ca = e->ar_ca; p.hd = e->ar_hd; p.y = e->ar_y; p.qc = e->ar_qc; p.part = e->ar_part;
    p.bar = e->ar_bar;
  }
  {
    // per image and step: 3 D^2 (self out, cross q, cross out) + 2 D Md (MLP) + C D (head) + attention dots
    const double macs = static_cast<double>(B) * L * (3.0 * D * D + 2.0 * D * e->Md + 1.0 * e->C * D + 2.0 * e->T * D);
    TimedScope ts(e, st, CAT_DEC_AR, 2.0 * macs);
    if (path == ArPath::Cluster) {
      PQ_TRY(dispatch_width(D, "dec_ar2", [&](auto w) {
        constexpr int W = decltype(w)::value;
        return e->ids_ld == 64 ? ar2_dispatch<W, 64>(e, q, st) : ar2_dispatch<W, 32>(e, q, st);
      }));
    } else {
      PQ_TRY(dispatch_width(D, "dec_ar", [&](auto w) {
        constexpr int W = decltype(w)::value;
        return dispatch_tokens(e->T, [&](auto tb) {
          return launch_k(e->lo, pq::dec_ar_kernel<W, decltype(tb)::value>, dim3(static_cast<unsigned>(e->lo.sm_count)),
                          dim3(pq::DEC_THREADS), pq::dec_ar_smem_bytes<W>(), st, p);
        });
      }));
    }
  }
  if (a->max_length < 0 && steps != nullptr) {
    PQ_TRY(launch_k(e->lo, pq::ar_steps_kernel, dim3(1), dim3(256), 0, st, static_cast<const int*>(e->ar_ids), e->ids_ld, B, L, 0,
                    steps));
    e->launches++;
  }
  return PARSEQ_OK;
}

// Cross-attention K/V of every decoder layer from the memory of the super-chunk's B images, once per image (the
// reference recomputes it in every decode call).
int cross_kv(parseq_engine* e, int B) {
  const int D = e->D, T = e->T;
  e->cur_cat = CAT_DEC_GEMM;
  for (int l = 0; l < e->cfg.dec_depth; ++l) {
    const std::string Ly = "decoder.layers." + std::to_string(l) + ".";
    const __nv_bfloat16* Wkv = e->wb(Ly + "cross_attn.in_proj_weight") + static_cast<long long>(D) * D;
    const float* bkv = e->wf(Ly + "cross_attn.in_proj_bias") + D;
    // stored column-blocked [2D/64][max_batch * T][64]: an image's K (V) panel of 64 channels is one contiguous T x 128 B
    // run - what a TMA box of the AR kernel and a head of the refine-pass attention read
    PQ_TRY(gemm(e, e->mem, D, Wkv, D, bkv, B * T, 2 * D, D, pq::EPI_BF16, 1.0f, nullptr, 0, 0,
                const_cast<__nv_bfloat16*>(ckv_of(e, l)), 2 * D, e->main, 1ll * e->max_batch * T));
  }
  return PARSEQ_OK;
}

// PARSeq: images [0, B) of a super-chunk -> e->mem, encoded in `chunk`-image pieces, and their cross K/V.  The kernel
// regime (fused GEMM + LayerNorm or not) follows the super-chunk, not `chunk`, so that the memory bits do not depend on
// `chunk` and every entry point (forward, score, beam search) reads the same memory of an image.
int encode_super(parseq_engine* e, const void* images, bool u8, int B) {
  for (int o = 0; o < B; o += e->chunk)
    PQ_TRY(encode_chunk(e, static_cast<const char*>(images) + o * image_bytes(e, u8), u8, std::min(B - o, e->chunk),
                        e->mem + 1ll * o * e->T * e->D, nullptr, e->main, true, B));
  return cross_kv(e, B);
}

// ViTSTR: the encoder blocks of images [0, B) in `chunk`-image pieces; after each piece, tail(o, Bs) runs on the final
// tokens of its images [o, o + Bs) (in e->x) - the norm and head of the kept rows.
template <typename Tail>
int vitstr_chunks(parseq_engine* e, const void* images, bool u8, int B, Tail&& tail) {
  for (int o = 0; o < B; o += e->chunk) {
    const int Bs = std::min(B - o, e->chunk);
    PQ_TRY(encode_chunk(e, static_cast<const char*>(images) + o * image_bytes(e, u8), u8, Bs, nullptr, nullptr, e->main, false));
    PQ_TRY(tail(o, Bs));
  }
  return PARSEQ_OK;
}

// n decoder groups, group i on stage i % stages: group(i, stage, stream).  With more than one stage in use the stages'
// streams run concurrently: each waits for `main`'s work so far, and `main` waits for all of them at the end (event
// fork / join, capturable into a CUDA graph).  Otherwise, and in timing mode (isolated kernel times), every group runs
// on `main`.
template <typename Group>
int fan_out(parseq_engine* e, int n, Group&& group) {
  const int ns = static_cast<int>(e->stages.size());
  const int used = std::min(n, ns);
  const bool fork = used > 1 && !e->timing;
  if (fork) {
    PQ_CUDA(cudaEventRecord(e->ev_enc, e->main));
    for (int s = 0; s < used; ++s) PQ_CUDA(cudaStreamWaitEvent(e->stages[static_cast<size_t>(s)].stream, e->ev_enc, 0));
  }
  for (int i = 0; i < n; ++i) {
    parseq_engine::Stage& sg = e->stages[static_cast<size_t>(i % ns)];
    PQ_TRY(group(i, sg, fork ? sg.stream : e->main));
  }
  if (fork) {
    for (int s = 0; s < used; ++s) {
      parseq_engine::Stage& sg = e->stages[static_cast<size_t>(s)];
      PQ_CUDA(cudaEventRecord(sg.ev_done, sg.stream));
      PQ_CUDA(cudaStreamWaitEvent(e->main, sg.ev_done, 0));
    }
  }
  return PARSEQ_OK;
}

// One super-chunk (B <= max_batch images): `main` encodes everything (in `chunk`-image pieces) and projects the cross
// K/V of the whole super-chunk; then the decoder - a latency-bound chain of small kernels - runs as ceil(B/dec_chunk)
// independent chains on their own streams, concurrently (fan_out).
// part 0: the whole super-chunk.  part 1 / 2 (host entry points, PARSeq only): the encoder of images [0, split) alone /
// the encoder of images [split, B) and everything after it - two graphs, so that the second half of the input is still
// uploading while the first half is being encoded.
// `mask`: the super-chunk's class allowlist rows (mask_ld words per image), or null.
int forward_super(parseq_engine* e, const parseq_forward_args* a, int b0, int B, int L, const void* images, bool u8,
                  float* logits, int* ids_out, int* steps, const uint32_t* mask, float* maps, int part = 0, int split = 0) {
  const int D = e->D, T = e->T;
  if (part == 1)
    return encode_chunk(e, images, u8, split, e->mem, nullptr, e->main, true, B);
  if (e->arch == 1) {               // ViTSTR: encoder blocks, then norm + head on the kept token rows of each chunk
    return vitstr_chunks(e, images, u8, B, [&](int o, int Bs) -> int {
      return vitstr_tail(e, Bs, L, logits + 1ll * o * L * e->C, ids_out ? ids_out + 1ll * o * L : nullptr,
                         mask ? mask + 1ll * o * e->mask_ld : nullptr, e->main);
    });
  }
  if (part == 2) {
    PQ_TRY(encode_chunk(e, static_cast<const char*>(images) + split * image_bytes(e, u8), u8, B - split,
                        e->mem + 1ll * split * T * D, nullptr, e->main, true, B));
    PQ_TRY(cross_kv(e, B));
  } else {
    PQ_TRY(encode_super(e, images, u8, B));
  }
  const ArPath path = ar_path(e);
  const bool ar_done = a->decode_ar && path != ArPath::Chain;
  e->ar_last_path = a->decode_ar ? static_cast<int>(path) : -1;
  if (ar_done) {
    PQ_TRY(ar_decode(e, path, a, b0, B, L, logits, steps, mask, e->main));
    if (a->refine_iters == 0) {      // nothing left for the chains but the final argmax (the AR kernels masked the logits)
      if (ids_out != nullptr) PQ_TRY(argmax_rows(e, logits, L, B, L, 0, ids_out, L, 0, nullptr, 0, nullptr, e->main));
      for (int o = 0; maps != nullptr && o < B; o += e->dec_chunk)
        PQ_TRY(ar_maps_pass(e, e->stages[static_cast<size_t>(o / e->dec_chunk)], o, std::min(B - o, e->dec_chunk), L,
                            e->ar_ids + 1ll * o * e->ids_ld, maps + 1ll * o * L * T, e->main));
      return PARSEQ_OK;
    }
  }
  // one decoder chain per dec_chunk images (B <= max_batch: one per stage at most)
  return fan_out(e, (B + e->dec_chunk - 1) / e->dec_chunk, [&](int s, parseq_engine::Stage& sg, cudaStream_t ds) -> int {
    const int o = s * e->dec_chunk;
    return decode_stage(e, sg, o, a, b0 + o, std::min(B - o, e->dec_chunk), L, logits + 1ll * o * L * e->C,
                        ids_out ? ids_out + 1ll * o * L : nullptr, steps, mask ? mask + 1ll * o * e->mask_ld : nullptr, ds,
                        ar_done, maps ? maps + 1ll * o * L * T : nullptr);
  });
}

int num_steps_of(const parseq_engine* e, int max_length) {
  const int ml = (max_length < 0) ? e->cfg.max_label_length
                                  : (max_length < e->cfg.max_label_length ? max_length : e->cfg.max_label_length);
  return ml + 1;
}

// Replays (capturing on first use) the CUDA graph of one super-chunk of Bc images on the static I/O buffers (a call with
// an allowlist: its rows are in e->in_mask).
int run_graph(parseq_engine* e, const parseq_forward_args* a, int Bc, int L, bool u8, int part = 0, int split = 0) {
  const bool masked = a->class_mask != nullptr;
  std::vector<int> key = {Bc, L, a->max_length < 0 ? 1 : 0, a->decode_ar ? 1 : 0, a->refine_iters, u8 ? 1 : 0, part, split,
                          masked ? 1 : 0};
  // the graphs of calls without maps keep their keys; part 1 (the first half's encoder) never touches the maps
  if (a->attn_maps != nullptr && part != 1) key.push_back(1);
  auto it = e->graphs.find(key);
  if (it == e->graphs.end()) {
    parseq_forward_args aa = *a;
    aa.batch = Bc;
    aa.forced_ids = nullptr;
    aa.forced_refine = nullptr;
    const long long before = e->launches;
    PQ_CUDA(cudaStreamBeginCapture(e->main, cudaStreamCaptureModeThreadLocal));
    int r = forward_super(e, &aa, 0, Bc, L, u8 ? static_cast<const void*>(e->in_images_u8) : static_cast<const void*>(e->in_images),
                          u8, e->out_logits, e->out_ids, e->out_steps, masked ? e->in_mask.get() : nullptr,
                          a->attn_maps != nullptr ? e->out_maps.get() : nullptr, part, split);
    cudaGraph_t g = nullptr;
    cudaError_t ce = cudaStreamEndCapture(e->main, &g);
    if (r != PARSEQ_OK) { if (g) cudaGraphDestroy(g); return r; }
    if (ce != cudaSuccess) return fail(PARSEQ_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(ce));
    cudaGraphExec_t exec = nullptr;
    ce = cudaGraphInstantiate(&exec, g, 0);
    cudaGraphDestroy(g);
    if (ce != cudaSuccess) return fail(PARSEQ_ERR_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(ce));
    parseq_engine::GraphEntry ge{GraphExec(exec), e->launches - before};
    e->launches = before;
    it = e->graphs.emplace(key, std::move(ge)).first;
  }
  PQ_CUDA(cudaGraphLaunch(it->second.exec, e->main));
  e->launches += it->second.kernels;
  return PARSEQ_OK;
}

// ---------------------------------------------------------------- raw crops of any size (crops.cuh)
// The crops of one parseq_forward_crops / parseq_forward_host_crops / parseq_resize_crops call, metadata validated.
struct CropBatch {
  const parseq_crops* c;
  bool host;                        // c->data is host memory: each super-chunk's bytes are staged in e->crop_stage
};

bool valid_rotation(int r) { return r == 0 || r == 90 || r == 180 || r == 270; }
// Crop i's rotation: its own (rotations) or the call's
int crop_rot(const parseq_crops* c, int i) { return c->rotations != nullptr ? c->rotations[i] : c->rotation; }

// The crop metadata, on the host alone (no handle or device needed).  These checks, and check_crop_smem, run before
// the first launch of a call: on failure nothing is enqueued.
int check_crops(int batch, const parseq_crops* c) {
  if (c == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (batch == 0) return PARSEQ_OK;
  if (c->data == nullptr || c->offsets == nullptr || c->sizes == nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "null crop data, offsets or sizes");
  if (c->rotations == nullptr && !valid_rotation(c->rotation))
    return fail(PARSEQ_ERR_INVALID_ARG, "rotation must be 0, 90, 180 or 270");
  for (int i = 0; i < batch; ++i) {
    if (c->rotations != nullptr && !valid_rotation(c->rotations[i]))
      return fail(PARSEQ_ERR_INVALID_ARG, "crop " + std::to_string(i) + ": rotation must be 0, 90, 180 or 270, got " +
                                              std::to_string(c->rotations[i]));
    const int h = c->sizes[2 * i], w = c->sizes[2 * i + 1];
    if (h < 1 || w < 1 || h > pq::CROP_MAX_SIDE || w > pq::CROP_MAX_SIDE)
      return fail(PARSEQ_ERR_INVALID_ARG, "crop " + std::to_string(i) + ": size " + std::to_string(h) + " x " +
                                              std::to_string(w) + ", sides must be in [1, 8192]");
    if (c->offsets[i] < 0 || c->offsets[i] > c->data_bytes - 3ll * h * w)
      return fail(PARSEQ_ERR_INVALID_ARG, "crop " + std::to_string(i) + ": offset + 3 h w exceeds data_bytes");
  }
  return PARSEQ_OK;
}

// The resize kernel's coefficient tables of every crop fit in shared memory (always at img_size 32 x 128 and 224 x 224).
int check_crop_smem(const parseq_engine* e, int batch, const parseq_crops* c) {
  int optin = 0;
  PQ_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->cfg.device));
  for (int i = 0; i < batch; ++i) {
    const int h = c->sizes[2 * i], w = c->sizes[2 * i + 1];
    const bool turn = crop_rot(c, i) == 90 || crop_rot(c, i) == 270;
    if (4ll * pq::crop_smem_ints(turn ? w : h, turn ? h : w, e->cfg.img_h, e->cfg.img_w) > optin)
      return fail(PARSEQ_ERR_UNSUPPORTED, "crop " + std::to_string(i) + ": resize tables exceed shared memory at this img_size");
  }
  return PARSEQ_OK;
}

// Crop i as the kernel reads it, rotated counter-clockwise by `rot` (np.rot90(crop, rot / 90)), its bytes at
// data + offsets[i] - base.
pq::CropDesc crop_desc(const parseq_crops* c, int i, long long base, int rot) {
  const int h = c->sizes[2 * i], w = c->sizes[2 * i + 1], row = 3 * w;
  const long long o = c->offsets[i] - base;
  switch (rot) {
    case 90: return pq::CropDesc{o + 3ll * (w - 1), -3, row, w, h};
    case 180: return pq::CropDesc{o + 1ll * row * (h - 1) + 3ll * (w - 1), -row, -3, h, w};
    case 270: return pq::CropDesc{o + 1ll * row * (h - 1), 3, -row, w, h};
    default: return pq::CropDesc{o, row, 3, h, w};
  }
}

// Bytes [lo, hi) of data that crops [i0, i1) occupy.
void crop_range(const parseq_crops* c, int i0, int i1, long long* lo, long long* hi) {
  *lo = c->offsets[i0];
  *hi = 0;
  for (int i = i0; i < i1; ++i) {
    const long long o = c->offsets[i];
    *lo = o < *lo ? o : *lo;
    const long long end = o + 3ll * c->sizes[2 * i] * c->sizes[2 * i + 1];
    *hi = end > *hi ? end : *hi;
  }
}

// Host crops: grows the staging buffer to the largest super-chunk of the call, before anything of the call is enqueued.
int crops_reserve(parseq_engine* e, const CropBatch& cb, int batch) {
  if (!cb.host) return PARSEQ_OK;
  long long need = 0;
  for (int b0 = 0; b0 < batch; b0 += e->max_batch) {
    long long lo, hi;
    crop_range(cb.c, b0, (batch - b0 < e->max_batch) ? batch : b0 + e->max_batch, &lo, &hi);
    need = hi - lo > need ? hi - lo : need;
  }
  return e->crop_stage.grow(e, need);
}

// Uploads the crop table of super-chunk [b0, b0 + Bc) on `st`.
int crops_table(parseq_engine* e, const CropBatch& cb, int b0, int Bc, cudaStream_t st) {
  long long lo = 0, hi = 0;
  if (cb.host) crop_range(cb.c, b0, b0 + Bc, &lo, &hi);
  e->crop_base = lo;
  e->crop_descs.resize(static_cast<size_t>(Bc));
  for (int i = 0; i < Bc; ++i) e->crop_descs[static_cast<size_t>(i)] = crop_desc(cb.c, b0 + i, lo, crop_rot(cb.c, b0 + i));
  // pageable source: the call returns once the table is staged, so crop_descs may change afterwards
  PQ_CUDA(cudaMemcpyAsync(e->crop_tab, e->crop_descs.data(), sizeof(pq::CropDesc) * Bc, cudaMemcpyHostToDevice, st));
  return PARSEQ_OK;
}

// Crops [b0 + i0, b0 + i1) of the super-chunk whose table is uploaded -> out [i1 - i0, img_h, img_w, 3] on `st` (host
// crops: their bytes are uploaded first, on the same stream).
int crops_resize(parseq_engine* e, const CropBatch& cb, int b0, int i0, int i1, uint8_t* out, cudaStream_t st) {
  const uint8_t* data = cb.c->data;
  if (cb.host) {
    long long lo, hi;
    crop_range(cb.c, b0 + i0, b0 + i1, &lo, &hi);
    PQ_CUDA(cudaMemcpyAsync(e->crop_stage + (lo - e->crop_base), data + lo, static_cast<size_t>(hi - lo), cudaMemcpyHostToDevice, st));
    data = e->crop_stage;
  }
  const int H = e->cfg.img_h, W = e->cfg.img_w;
  int smem = 0;
  for (int i = i0; i < i1; ++i) {
    const pq::CropDesc& d = e->crop_descs[static_cast<size_t>(i)];
    const int s = 4 * pq::crop_smem_ints(d.h, d.w, H, W);
    smem = s > smem ? s : smem;
  }
  const int lines = H > W ? H : W;          // second-pass lines: out_h, or out_w for tall crops
  const dim3 grid((lines + pq::CROP_BAND - 1) / pq::CROP_BAND, i1 - i0);
  TimedScope ts(e, st, CAT_MISC, 0.0);
  // no PDL: the kernel reads what the copies and the previous forward left behind
  return launch_ex(LaunchConfig(grid, dim3(pq::CROP_THREADS), static_cast<size_t>(smem), st, 0, false),
                   pq::crop_resize_bicubic_kernel, data, static_cast<const pq::CropDesc*>(e->crop_tab + i0), H, W,
                   out + 3ll * H * W * i0);
}

// Shared checks of the forward entry points of raw crops; teacher forcing is a float-input debug feature.
int check_crops_call(parseq_engine* e, const parseq_forward_args* a, const parseq_crops* crops, const float* logits) {
  if (a == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (a->batch < 0 || a->refine_iters < 0) return fail(PARSEQ_ERR_INVALID_ARG, "negative batch / refine_iters");
  if (a->forced_ids != nullptr || a->forced_refine != nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "teacher forcing is a device-pointer API (parseq_forward)");
  PQ_TRY(check_crops(a->batch, crops));
  if (logits == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  return check_crop_smem(e, a->batch, crops);
}

// ---------------------------------------------------------------- text regions of full frames (regions.cuh)
// The metadata of a parseq_warp_regions call, on the host alone (no handle or device needed), before anything is
// enqueued.  *packed: the bytes of all rectified crops, sum of 3 h w.
// The frames of a region call, and region i's frame index and crop size; the checks parseq_warp_regions and
// parseq_warp_polygons share.
int check_region_frames(int64_t frames_bytes, const int64_t* frame_offsets, const int32_t* frame_sizes, int num_frames) {
  if (num_frames < 1) return fail(PARSEQ_ERR_INVALID_ARG, "num_frames must be >= 1");
  for (int f = 0; f < num_frames; ++f) {
    const int H = frame_sizes[2 * f], W = frame_sizes[2 * f + 1];
    if (H < 1 || W < 1 || H > pq::REGION_MAX_FRAME_SIDE || W > pq::REGION_MAX_FRAME_SIDE)
      return fail(PARSEQ_ERR_INVALID_ARG, "frame " + std::to_string(f) + ": size " + std::to_string(H) + " x " +
                                              std::to_string(W) + ", sides must be in [1, 32768]");
    if (frame_offsets[f] < 0 || frame_offsets[f] > frames_bytes - 3ll * H * W)
      return fail(PARSEQ_ERR_INVALID_ARG, "frame " + std::to_string(f) + ": offset + 3 H W exceeds frames_bytes");
  }
  return PARSEQ_OK;
}

int check_region_crop(const std::string& at, const int32_t* frame_index, const int32_t* sizes, int num_frames, int i) {
  if (frame_index[i] < 0 || frame_index[i] >= num_frames)
    return fail(PARSEQ_ERR_INVALID_ARG, at + "frame_index " + std::to_string(frame_index[i]) + " out of range");
  const int h = sizes[2 * i], w = sizes[2 * i + 1];
  if (h < 1 || w < 1 || h > pq::REGION_MAX_SIDE || w > pq::REGION_MAX_SIDE)
    return fail(PARSEQ_ERR_INVALID_ARG, at + "size " + std::to_string(h) + " x " + std::to_string(w) +
                                            ", sides must be in [1, 8192]");
  return PARSEQ_OK;
}

int check_regions(int count, const parseq_regions* r, const uint8_t* out, long long out_bytes, long long* packed) {
  if (r == nullptr || count < 0) return fail(PARSEQ_ERR_INVALID_ARG, "null argument or negative count");
  *packed = 0;
  if (count == 0) return PARSEQ_OK;
  if (r->frames == nullptr || r->frame_offsets == nullptr || r->frame_sizes == nullptr || r->frame_index == nullptr ||
      r->sizes == nullptr || r->coeffs == nullptr || out == nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "null frames, frame_offsets, frame_sizes, frame_index, sizes, coeffs or out");
  PQ_TRY(check_region_frames(r->frames_bytes, r->frame_offsets, r->frame_sizes, r->num_frames));
  for (int i = 0; i < count; ++i) {
    const std::string at = "region " + std::to_string(i) + ": ";
    PQ_TRY(check_region_crop(at, r->frame_index, r->sizes, r->num_frames, i));
    const int h = r->sizes[2 * i], w = r->sizes[2 * i + 1];
    const double* a = r->coeffs + 8ll * i;
    for (int k = 0; k < 8; ++k)
      if (!std::isfinite(a[k])) return fail(PARSEQ_ERR_INVALID_ARG, at + "non-finite coefficient");
    // the denominator is affine in the output point: positive at the four corner pixel centres, it is positive at
    // every pixel centre, so the kernel's divisions never meet 0 or a sign change
    for (int k = 0; k < 4; ++k) {
      const double xin = (k & 1) ? w - 0.5 : 0.5, yin = (k & 2) ? h - 0.5 : 0.5;
      if (!(a[6] * xin + a[7] * yin + 1.0 > 0.0))
        return fail(PARSEQ_ERR_INVALID_ARG, at + "the map's denominator a6 x + a7 y + 1 is not positive at a corner");
    }
    *packed += 3ll * h * w;
  }
  if (out_bytes < *packed)
    return fail(PARSEQ_ERR_INVALID_ARG, "out_bytes (" + std::to_string(out_bytes) + ") is smaller than the packed crops (" +
                                            std::to_string(*packed) + ")");
  return PARSEQ_OK;
}

// ---------------------------------------------------------------- curved regions: thin-plate splines (regions.cuh)
// TRBA's GridGenerator (RARE's TPS) with F = 2k fiducials C at C_x = numpy.linspace(-1, 1, k), C_y = -1 (top) and +1
// (bottom).  delta_C [F + 3][F + 3] is _build_inv_delta_C's matrix: rows m < F are (1, C_x[m], C_y[m], hat_C[m][.]) with
// hat_C = r^2 ln r off the diagonal and 0 on it, then the rows (0, 0, 0, C_x), (0, 0, 0, C_y) and (0, 0, 0, 1).  Its
// inverse depends only on k: it is computed once per k by Gauss-Jordan elimination with partial pivoting (first
// largest pivot in row order) and kept for the process.  The library is built with -ffp-contract=off, so the host
// arithmetic here is one rounding per operation on every host compiler.

// numpy.linspace(-1, 1, k) bit for bit: j * (2 / (k - 1)) + (-1), the last point exactly 1
void tps_cx(int k, double* cx) {
  const double step = 2.0 / static_cast<double>(k - 1);
  for (int j = 0; j < k - 1; ++j) cx[j] = static_cast<double>(j) * step + (-1.0);
  cx[k - 1] = 1.0;
}

const std::vector<double>& tps_inv_delta_c(int k) {
  static std::mutex mu;
  static std::map<int, std::vector<double>> cache;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(k);
  if (it != cache.end()) return it->second;
  const int F = 2 * k, n = F + 3;
  double cx[pq::TPS_MAX_K];
  tps_cx(k, cx);
  std::vector<double> a(static_cast<size_t>(n) * n, 0.0), inv(static_cast<size_t>(n) * n, 0.0);
  auto fx = [&](int m) { return cx[m % k]; };
  auto fy = [&](int m) { return m < k ? -1.0 : 1.0; };
  for (int i = 0; i < F; ++i) {
    a[i * n + 0] = 1.0;
    a[i * n + 1] = fx(i);
    a[i * n + 2] = fy(i);
    for (int j = 0; j < F; ++j) {
      if (i == j) continue;
      const double dx = fx(i) - fx(j), dy = fy(i) - fy(j);
      const double r = std::sqrt(dx * dx + dy * dy);
      a[i * n + 3 + j] = (r * r) * std::log(r);
    }
    a[(F + 0) * n + 3 + i] = fx(i);
    a[(F + 1) * n + 3 + i] = fy(i);
    a[(F + 2) * n + 3 + i] = 1.0;
  }
  for (int i = 0; i < n; ++i) inv[i * n + i] = 1.0;
  for (int c = 0; c < n; ++c) {
    int piv = c;
    for (int r = c + 1; r < n; ++r)
      if (std::fabs(a[r * n + c]) > std::fabs(a[piv * n + c])) piv = r;
    if (piv != c)
      for (int j = 0; j < n; ++j) {
        std::swap(a[c * n + j], a[piv * n + j]);
        std::swap(inv[c * n + j], inv[piv * n + j]);
      }
    const double p = a[c * n + c];
    for (int j = 0; j < n; ++j) {
      a[c * n + j] /= p;
      inv[c * n + j] /= p;
    }
    for (int r = 0; r < n; ++r) {
      const double f = a[r * n + c];
      if (r == c || f == 0.0) continue;
      for (int j = 0; j < n; ++j) {
        a[r * n + j] -= f * a[c * n + j];
        inv[r * n + j] -= f * inv[c * n + j];
      }
    }
  }
  return cache.emplace(k, std::move(inv)).first->second;
}

// T [F + 3][2] = inv_delta_C [F + 3][F + 3] . [C'; 0], summed in index order; points: C' [F][2], engine order.
void tps_solve(int k, const double* points, double* coeffs) {
  const std::vector<double>& inv = tps_inv_delta_c(k);
  const int F = 2 * k, n = F + 3;
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < 2; ++c) {
      double acc = 0.0;
      for (int j = 0; j < F; ++j) acc += inv[static_cast<size_t>(i) * n + j] * points[2 * j + c];
      coeffs[2 * i + c] = acc;
    }
}

int check_polygon_points(const std::string& at, int num_points, const double* points) {
  if (num_points % 2 != 0 || num_points < 2 * pq::TPS_MIN_K || num_points > 2 * pq::TPS_MAX_K)
    return fail(PARSEQ_ERR_INVALID_ARG, at + std::to_string(num_points) + " points, a polygon needs an even count in [6, 64]");
  for (int j = 0; j < 2 * num_points; ++j)
    if (!std::isfinite(points[j])) return fail(PARSEQ_ERR_INVALID_ARG, at + "non-finite point");
  return PARSEQ_OK;
}

// The metadata of a parseq_warp_polygons call, on the host alone (no handle or device needed), before anything is
// enqueued.  *packed: the bytes of all rectified crops, sum of 3 h w.
int check_polygons(int count, const parseq_polygons* r, const uint8_t* out, long long out_bytes, long long* packed) {
  if (r == nullptr || count < 0) return fail(PARSEQ_ERR_INVALID_ARG, "null argument or negative count");
  *packed = 0;
  if (count == 0) return PARSEQ_OK;
  if (r->frames == nullptr || r->frame_offsets == nullptr || r->frame_sizes == nullptr || r->frame_index == nullptr ||
      r->sizes == nullptr || r->num_points == nullptr || r->points == nullptr || out == nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "null frames, frame_offsets, frame_sizes, frame_index, sizes, num_points, points or out");
  PQ_TRY(check_region_frames(r->frames_bytes, r->frame_offsets, r->frame_sizes, r->num_frames));
  long long first = 0;                     // the region's first point in `points`
  for (int i = 0; i < count; ++i) {
    const std::string at = "region " + std::to_string(i) + ": ";
    PQ_TRY(check_region_crop(at, r->frame_index, r->sizes, r->num_frames, i));
    PQ_TRY(check_polygon_points(at, r->num_points[i], r->points + 2 * first));
    first += r->num_points[i];
    *packed += 3ll * r->sizes[2 * i] * r->sizes[2 * i + 1];
  }
  if (out_bytes < *packed)
    return fail(PARSEQ_ERR_INVALID_ARG, "out_bytes (" + std::to_string(out_bytes) + ") is smaller than the packed crops (" +
                                            std::to_string(*packed) + ")");
  return PARSEQ_OK;
}

// The causal masks of every row count P (scoring, and the map pass of AR-only schedules), on first use.
int causal_reserve(parseq_engine* e) {
  if (e->sc_causal != nullptr) return PARSEQ_OK;
  const int L = e->L;
  // the canonical left-to-right permutation (system.py:153-167): query i and content row i see keys 0..i
  std::vector<unsigned char> h(static_cast<size_t>(L) * L * L, 0);
  for (int P = 1; P <= L; ++P)
    for (int q = 0; q < P; ++q)
      for (int k = 0; k < P; ++k) h[static_cast<size_t>(P - 1) * L * L + static_cast<size_t>(q) * P + k] = k > q ? 1 : 0;
  PQ_TRY(e->sc_causal.alloc(static_cast<long long>(h.size())));
  PQ_CUDA(cudaMemcpy(e->sc_causal, h.data(), h.size(), cudaMemcpyHostToDevice));
  return PARSEQ_OK;
}

// Cross-attention map buffers, on the first call that asks for maps: the static maps the graphs write, and the causal
// masks only for an AR-only schedule (the one whose map pass reads them).
int maps_reserve(parseq_engine* e, const parseq_forward_args* a) {
  PQ_TRY(e->out_maps.reserve(1ll * e->max_batch * e->L * e->T));
  return a->decode_ar && a->refine_iters == 0 ? causal_reserve(e) : PARSEQ_OK;
}

// Common driver of parseq_forward / parseq_forward_host. `host` selects H2D/D2H vs D2D staging copies.
// `crops` (raw crops of any size, u8): each super-chunk is resized into the static uint8 input in place of the copy.
int forward_impl(parseq_engine* e, const parseq_forward_args* a, const void* images_any, float* logits, int32_t* ids,
                 int32_t* steps, cudaStream_t user, bool host, bool u8 = false, const CropBatch* crops = nullptr) {
  if (a->class_mask != nullptr && (a->forced_ids != nullptr || a->forced_refine != nullptr))
    return fail(PARSEQ_ERR_INVALID_ARG, "class_mask cannot be combined with teacher forcing");
  float* const maps = a->attn_maps;
  if (maps != nullptr) {
    if (e->arch != 0) return fail(PARSEQ_ERR_UNSUPPORTED, "attn_maps: ViTSTR has no decoder cross-attention");
    if (a->forced_ids != nullptr || a->forced_refine != nullptr)
      return fail(PARSEQ_ERR_INVALID_ARG, "attn_maps cannot be combined with teacher forcing");
    PQ_TRY(maps_reserve(e, a));
  }
  const int L = num_steps_of(e, a->max_length);
  const bool testing = a->max_length < 0;
  const long long img_sz = image_bytes(e, u8);
  const char* images = static_cast<const char*>(images_any);
  void* in_static = u8 ? static_cast<void*>(e->in_images_u8) : static_cast<void*>(e->in_images);
  const bool eager = !e->use_graph || e->timing || a->forced_ids != nullptr || a->forced_refine != nullptr;
  const cudaMemcpyKind kin = host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  const cudaMemcpyKind kout = host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  // the allowlist rows of super-chunk [b0, b0 + Bc) -> the static rows the graphs read (on `main`: after the previous
  // super-chunk's graph has read them); nothing at all for a call without one
  const long long mask_row_bytes = 4ll * e->mask_ld;
  auto stage_mask = [&](int b0, int Bc) -> int {
    if (a->class_mask == nullptr) return PARSEQ_OK;
    PQ_CUDA(cudaMemcpyAsync(e->in_mask, a->class_mask + 1ll * b0 * e->mask_ld, static_cast<size_t>(Bc * mask_row_bytes), kin,
                            e->main));
    return PARSEQ_OK;
  };
  // the static maps of super-chunk [b0, b0 + Bc) -> the caller's, as the logits
  auto copy_maps = [&](int b0, int Bc) -> int {
    if (maps == nullptr) return PARSEQ_OK;
    PQ_CUDA(cudaMemcpyAsync(maps + 1ll * b0 * L * e->T, e->out_maps, static_cast<size_t>(1ll * Bc * L * e->T) * 4, kout, e->main));
    return PARSEQ_OK;
  };
  PQ_TRY(enter_main(e, user));
  PQ_TRY(launch_k(e->lo, pq::set_int_kernel, dim3(1), dim3(32), 0, e->main, e->out_steps,
                  (testing && a->decode_ar && e->arch == 0) ? 0 : L));
  e->launches++;
  for (int b0 = 0; b0 < a->batch; b0 += e->max_batch) {
    const int Bc = (a->batch - b0 < e->max_batch) ? (a->batch - b0) : e->max_batch;
    if (eager && !host) {
      const char* in = reinterpret_cast<const char*>(e->in_images_u8.get());
      if (crops) {
        PQ_TRY(crops_table(e, *crops, b0, Bc, e->main));
        PQ_TRY(crops_resize(e, *crops, b0, 0, Bc, e->in_images_u8, e->main));
      } else {
        in = images + b0 * img_sz;
      }
      PQ_TRY(forward_super(e, a, b0, Bc, L, in, u8, logits + 1ll * b0 * L * e->C, ids ? ids + 1ll * b0 * L : nullptr,
                           e->out_steps, a->class_mask ? a->class_mask + 1ll * b0 * e->mask_ld : nullptr,
                           maps ? maps + 1ll * b0 * L * e->T : nullptr));
      continue;
    }
    if (host && !eager && e->arch == 0 && Bc >= 256 && e->chunk >= Bc) {
      // upload in two halves on the copy stream; the encoder of the first half (its own graph) runs under the second upload
      const int split = ((Bc / 2 + 7) / 8) * 8;
      PQ_CUDA(cudaEventRecord(e->ev_c[2], e->main));                       // previous work on `main` (and the caller's stream)
      PQ_CUDA(cudaStreamWaitEvent(e->copy, e->ev_c[2], 0));
      if (crops) {
        PQ_TRY(crops_table(e, *crops, b0, Bc, e->copy));
        PQ_TRY(crops_resize(e, *crops, b0, 0, split, e->in_images_u8, e->copy));
      } else {
        PQ_CUDA(cudaMemcpyAsync(in_static, images + b0 * img_sz, static_cast<size_t>(split * img_sz), kin, e->copy));
      }
      PQ_CUDA(cudaEventRecord(e->ev_c[0], e->copy));
      if (crops) {
        PQ_TRY(crops_resize(e, *crops, b0, split, Bc, e->in_images_u8, e->copy));
      } else {
        PQ_CUDA(cudaMemcpyAsync(static_cast<char*>(in_static) + split * img_sz, images + (b0 + split) * img_sz,
                                static_cast<size_t>((Bc - split) * img_sz), kin, e->copy));
      }
      PQ_CUDA(cudaEventRecord(e->ev_c[1], e->copy));
      PQ_TRY(stage_mask(b0, Bc));
      PQ_CUDA(cudaStreamWaitEvent(e->main, e->ev_c[0], 0));
      PQ_TRY(run_graph(e, a, Bc, L, u8, 1, split));
      PQ_CUDA(cudaStreamWaitEvent(e->main, e->ev_c[1], 0));
      PQ_TRY(run_graph(e, a, Bc, L, u8, 2, split));
      PQ_CUDA(cudaMemcpyAsync(logits + 1ll * b0 * L * e->C, e->out_logits, static_cast<size_t>(1ll * Bc * L * e->C) * 4, kout,
                              e->main));
      if (ids) PQ_CUDA(cudaMemcpyAsync(ids + 1ll * b0 * L, e->out_ids, static_cast<size_t>(1ll * Bc * L) * 4, kout, e->main));
      PQ_TRY(copy_maps(b0, Bc));
      continue;
    }
    if (crops) {
      PQ_TRY(crops_table(e, *crops, b0, Bc, e->main));
      PQ_TRY(crops_resize(e, *crops, b0, 0, Bc, e->in_images_u8, e->main));
    } else {
      PQ_CUDA(cudaMemcpyAsync(in_static, images + b0 * img_sz, static_cast<size_t>(Bc * img_sz), kin, e->main));
    }
    PQ_TRY(stage_mask(b0, Bc));
    if (eager) {
      PQ_TRY(forward_super(e, a, b0, Bc, L, in_static, u8, e->out_logits, e->out_ids, e->out_steps,
                           a->class_mask ? e->in_mask.get() : nullptr, maps ? e->out_maps.get() : nullptr));
    } else {
      PQ_TRY(run_graph(e, a, Bc, L, u8));
    }
    PQ_CUDA(cudaMemcpyAsync(logits + 1ll * b0 * L * e->C, e->out_logits, static_cast<size_t>(1ll * Bc * L * e->C) * 4, kout,
                            e->main));
    if (ids) PQ_CUDA(cudaMemcpyAsync(ids + 1ll * b0 * L, e->out_ids, static_cast<size_t>(1ll * Bc * L) * 4, kout, e->main));
    PQ_TRY(copy_maps(b0, Bc));
  }
  if (steps) PQ_CUDA(cudaMemcpyAsync(steps, e->out_steps, 4, kout, e->main));
  return leave_main(e, user);
}

// parseq_forward / _host / _u8 / _host_u8: `host` (host buffers; the call returns once the outputs are there) and `u8`
// (uint8 HWC images) as in forward_impl.  Teacher forcing is a device-pointer API.
int forward_call(parseq_engine* e, const parseq_forward_args* a, const void* images, float* logits, int32_t* ids,
                 int32_t* steps, parseq_stream_t stream, bool host, bool u8) {
  if (a == nullptr || images == nullptr || logits == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  if (a->batch < 0 || a->refine_iters < 0) return fail(PARSEQ_ERR_INVALID_ARG, "negative batch / refine_iters");
  if (a->batch == 0) return PARSEQ_OK;
  if (host && (a->forced_ids != nullptr || a->forced_refine != nullptr))
    return fail(PARSEQ_ERR_INVALID_ARG, "teacher forcing is a device-pointer API (parseq_forward)");
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  PQ_TRY(forward_impl(e, a, images, logits, ids, steps, reinterpret_cast<cudaStream_t>(stream), host, u8));
  if (host) PQ_CUDA(cudaStreamSynchronize(e->main));
  return PARSEQ_OK;
}

// ---------------------------------------------------------------- orientation search (parseq_forward_crops_oriented)
// The orientation arguments, on the host alone (no handle or device needed).
int check_orient(const parseq_orient_args* o) {
  if (o == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  const int R = o->num_orientations;
  if (R < 1 || R > 4) return fail(PARSEQ_ERR_INVALID_ARG, "num_orientations must be in [1, 4], got " + std::to_string(R));
  for (int r = 0; r < R; ++r) {
    if (!valid_rotation(o->orientations[r]))
      return fail(PARSEQ_ERR_INVALID_ARG, "orientations must be 0, 90, 180 or 270, got " + std::to_string(o->orientations[r]));
    for (int q = 0; q < r; ++q)
      if (o->orientations[q] == o->orientations[r])
        return fail(PARSEQ_ERR_INVALID_ARG, "orientations must be distinct, " + std::to_string(o->orientations[r]) + " repeats");
  }
  if (o->rotation_out == nullptr || o->confidence_out == nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "null rotation_out or confidence_out");
  return PARSEQ_OK;
}

// Pass 1 over all crops at o_0 (forward_impl), the confidence kernel, the list of crops to re-read (with a threshold:
// after the call's one host synchronisation), then pass 2 in super-chunks of whole crops, each followed by the select
// kernel.  `c`: the crops at rotation o_0; `host`: their bytes are in host memory, staged in e->crop_stage per pass-1
// super-chunk and per pass-2 super-chunk (which packs its listed crops one after another).
int orient_impl(parseq_engine* e, const parseq_forward_args* a, const parseq_crops& c, bool host, const parseq_orient_args* o,
                float* logits, int32_t* ids, int32_t* steps, cudaStream_t user) {
  const int N = a->batch, R = o->num_orientations, R1 = R - 1;
  const int L = num_steps_of(e, a->max_length);
  const bool testing = a->max_length < 0;
  // the rows past the step count are dropped with the shape (forward returns [N, S, C]) only here
  const bool zero_tail = testing && a->decode_ar && a->refine_iters == 0 && e->arch == 0;
  float* const maps = a->attn_maps;
  PQ_TRY(e->or_rd.reserve(e->max_batch));
  PQ_TRY(e->or_steps.reserve(1));
  PQ_TRY(e->or_conf.reserve(e->max_batch));
  const CropBatch cb{&c, host};
  PQ_TRY(forward_impl(e, a, nullptr, logits, ids, nullptr, user, false, true, &cb));
  PQ_TRY(enter_main(e, user));
  {
    TimedScope ts(e, e->main, CAT_ORIENT, 0.0);
    PQ_TRY(launch_ex(LaunchConfig(dim3(N), dim3(pq::ORIENT_THREADS), 0, e->main, 0, false), pq::orient_init_kernel, logits,
                     static_cast<int*>(ids), maps, L, e->C, e->T, o->orientations[0], static_cast<const int*>(e->out_steps),
                     zero_tail, static_cast<int*>(e->or_steps), static_cast<int*>(o->rotation_out), o->confidence_out));
  }
  std::vector<int> list;
  if (R > 1) {
    if (std::isnan(o->min_confidence)) {
      list.resize(static_cast<size_t>(N));
      for (int b = 0; b < N; ++b) list[static_cast<size_t>(b)] = b;
    } else {
      std::vector<float> c0(static_cast<size_t>(N));
      PQ_CUDA(cudaMemcpyAsync(c0.data(), o->confidence_out, 4ull * N, cudaMemcpyDeviceToHost, e->main));
      PQ_CUDA(cudaStreamSynchronize(e->main));
      for (int b = 0; b < N; ++b)
        if (!(c0[static_cast<size_t>(b)] >= o->min_confidence)) list.push_back(b);
    }
  }
  e->orient_rereads = static_cast<long long>(list.size());
  e->orient_readings = 0;
  const bool eager = !e->use_graph || e->timing;
  pq::OrientList rest{{0, 0, 0, 0}};
  for (int r = 1; r < R; ++r) rest.o[r - 1] = o->orientations[r];
  const int per = R1 > 0 ? e->max_batch / R1 : 0;        // whole crops per pass-2 super-chunk
  std::vector<int> rd;
  std::vector<int64_t> poff;
  std::vector<int32_t> psz;
  for (size_t k0 = 0; k0 < list.size(); k0 += static_cast<size_t>(per)) {
    const int nk = static_cast<int>(std::min(list.size() - k0, static_cast<size_t>(per)));
    const int n = nk * R1;
    int nb = 1;                                            // a power of two (or max_batch): few distinct graphs
    while (nb < n) nb <<= 1;
    nb = std::min(nb, e->max_batch);
    e->orient_readings += nb;
    rd.resize(static_cast<size_t>(nb));
    e->crop_descs.resize(static_cast<size_t>(nb));
    e->crop_base = 0;
    parseq_crops pc = c;                                   // the crops the super-chunk's table points into
    if (host) {
      poff.resize(static_cast<size_t>(nk));
      psz.resize(2 * static_cast<size_t>(nk));
      long long off = 0;
      for (int k = 0; k < nk; ++k) {
        const int b = list[k0 + static_cast<size_t>(k)];
        const long long bytes = 3ll * c.sizes[2 * b] * c.sizes[2 * b + 1];
        PQ_CUDA(cudaMemcpyAsync(e->crop_stage + off, c.data + c.offsets[b], static_cast<size_t>(bytes), cudaMemcpyHostToDevice,
                                e->main));
        poff[static_cast<size_t>(k)] = off;
        psz[2 * static_cast<size_t>(k)] = c.sizes[2 * b];
        psz[2 * static_cast<size_t>(k) + 1] = c.sizes[2 * b + 1];
        off += bytes;
      }
      pc.data = e->crop_stage;
      pc.data_bytes = off;
      pc.offsets = poff.data();
      pc.sizes = psz.data();
    }
    for (int j = 0; j < nb; ++j) {
      const int jj = std::min(j, n - 1);                   // padding: copies of the last reading
      const int k = jj / R1;
      const int b = list[k0 + static_cast<size_t>(k)];
      rd[static_cast<size_t>(j)] = b;
      e->crop_descs[static_cast<size_t>(j)] = crop_desc(&pc, host ? k : b, 0, rest.o[jj % R1]);
    }
    // pageable sources: the calls return once the tables are staged, so rd and crop_descs may change afterwards
    PQ_CUDA(cudaMemcpyAsync(e->or_rd, rd.data(), 4ull * nb, cudaMemcpyHostToDevice, e->main));
    PQ_CUDA(cudaMemcpyAsync(e->crop_tab, e->crop_descs.data(), sizeof(pq::CropDesc) * nb, cudaMemcpyHostToDevice, e->main));
    PQ_TRY(launch_k(e->lo, pq::set_int_kernel, dim3(1), dim3(32), 0, e->main, static_cast<int*>(e->out_steps),
                    (testing && a->decode_ar && e->arch == 0) ? 0 : L));
    e->launches++;
    PQ_TRY(crops_resize(e, CropBatch{&pc, false}, 0, 0, nb, e->in_images_u8, e->main));
    if (a->class_mask != nullptr) {
      TimedScope ts(e, e->main, CAT_ORIENT, 0.0);
      PQ_TRY(launch_ex(LaunchConfig(dim3((nb * e->mask_ld + 255) / 256), dim3(256), 0, e->main, 0, false),
                       pq::gather_rows_kernel, a->class_mask, static_cast<const int*>(e->or_rd), nb, e->mask_ld,
                       static_cast<uint32_t*>(e->in_mask)));
    }
    parseq_forward_args a2 = *a;
    a2.batch = nb;
    if (eager) {
      PQ_TRY(forward_super(e, &a2, 0, nb, L, e->in_images_u8, true, e->out_logits, e->out_ids, e->out_steps,
                           a->class_mask ? e->in_mask.get() : nullptr, maps ? e->out_maps.get() : nullptr));
    } else {
      PQ_TRY(run_graph(e, &a2, nb, L, true));
    }
    {
      TimedScope ts(e, e->main, CAT_ORIENT, 0.0);
      PQ_TRY(launch_ex(LaunchConfig(dim3(n), dim3(pq::ORIENT_THREADS), 0, e->main, 0, false), pq::orient_conf_kernel,
                       static_cast<const float*>(e->out_logits), L, e->C, static_cast<float*>(e->or_conf)));
    }
    TimedScope ts(e, e->main, CAT_ORIENT, 0.0);
    PQ_TRY(launch_ex(LaunchConfig(dim3(nk), dim3(pq::ORIENT_THREADS), 0, e->main, 0, false), pq::orient_select_kernel,
                     static_cast<const float*>(e->out_logits), static_cast<const int*>(e->out_ids),
                     static_cast<const float*>(maps ? e->out_maps.get() : nullptr), static_cast<const float*>(e->or_conf),
                     static_cast<const int*>(e->or_rd), R1, rest, L, e->C, e->T, static_cast<const int*>(e->out_steps), zero_tail,
                     static_cast<int*>(e->or_steps), logits, static_cast<int*>(ids), maps,
                     static_cast<int*>(o->rotation_out), o->confidence_out));
  }
  if (steps) PQ_CUDA(cudaMemcpyAsync(steps, e->or_steps, 4, cudaMemcpyDeviceToDevice, e->main));
  return leave_main(e, user);
}

// ---------------------------------------------------------------- candidate scoring (parseq_score)
// The metadata of a score call, on the host alone (no handle or device needed).  max_label_length < 0: the counts only.
// Target row m (pitch max_label_length + 1) holds c_1..c_n (head classes 1..C-1) and EOS (0) at position n.
int check_score(const parseq_score_args* a, int max_label_length, int num_classes) {
  if (a == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (a->batch < 0 || a->num_candidates < 0) return fail(PARSEQ_ERR_INVALID_ARG, "negative batch / num_candidates");
  if (a->batch == 0) return a->num_candidates == 0 ? PARSEQ_OK : fail(PARSEQ_ERR_INVALID_ARG, "candidates without images");
  if (a->per_image == nullptr || a->targets == nullptr || a->lengths == nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "null per_image, targets or lengths");
  long long sum = 0;
  for (int b = 0; b < a->batch; ++b) {
    if (a->per_image[b] < 1) return fail(PARSEQ_ERR_INVALID_ARG, "image " + std::to_string(b) + ": per_image must be >= 1");
    sum += a->per_image[b];
  }
  if (sum != a->num_candidates)
    return fail(PARSEQ_ERR_INVALID_ARG, "per_image sums to " + std::to_string(sum) + ", num_candidates is " +
                                            std::to_string(a->num_candidates));
  if (max_label_length < 0) return PARSEQ_OK;
  const int L = max_label_length + 1, C = num_classes;
  for (int m = 0; m < a->num_candidates; ++m) {
    const std::string who = "candidate " + std::to_string(m) + ": ";
    const int n = a->lengths[m];
    if (n < 0 || n > max_label_length)
      return fail(PARSEQ_ERR_INVALID_ARG, who + "length " + std::to_string(n) + " outside [0, max_label_length = " +
                                              std::to_string(max_label_length) + "]");
    const int32_t* t = a->targets + 1ll * m * L;
    for (int i = 0; i < n; ++i) {
      if (t[i] == 0) return fail(PARSEQ_ERR_INVALID_ARG, who + "EOS at position " + std::to_string(i) + ", before its end " + std::to_string(n));
      if (t[i] == C || t[i] == C + 1) return fail(PARSEQ_ERR_INVALID_ARG, who + "BOS or PAD id at position " + std::to_string(i));
      if (t[i] < 1 || t[i] > C + 1)
        return fail(PARSEQ_ERR_INVALID_ARG, who + "id " + std::to_string(t[i]) + " at position " + std::to_string(i) +
                                                " outside the character classes [1, " + std::to_string(C - 1) + "]");
    }
    if (t[n] != 0) return fail(PARSEQ_ERR_INVALID_ARG, who + "no EOS (0) at position n = " + std::to_string(n));
  }
  return PARSEQ_OK;
}

// Scoring buffers, on the first score call (an engine that never scores allocates none of them): the chains' LSE
// partials and target logits (PARSeq), ViTSTR's partials of a chunk, and the causal masks of every row count P.
int score_reserve(parseq_engine* e) {
  const int L = e->L;
  const long long ntiles = (e->C + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
  const long long Rd = 1ll * e->dec_chunk * L;
  if (e->arch == 0) {
    for (auto& sg : e->stages) {
      PQ_TRY(sg.lse_part.reserve(Rd * ntiles));
      PQ_TRY(sg.lse_tlogit.reserve(Rd));
    }
    PQ_TRY(causal_reserve(e));
  } else {
    PQ_TRY(e->sc_vt_part.reserve(1ll * e->chunk * L * ntiles));
  }
  return PARSEQ_OK;
}

// A group of candidates decoded in one pass of a chain: candidates [m0, m1) of images [b_lo, b_lo + nimg), P rows each
// (P = the longest label + 1), at most dec_chunk * L rows.  Offsets index the call's metadata (ints).
struct ScoreGroup {
  int m0, m1, P, b_lo, nimg, max_rows;
  long long ids_off, tgt_off, cand_off;
};

// Scores candidate labels of a batch of images (parseq_score): encoder and cross K/V once per super-chunk, then the
// candidates of its images in groups over the chains (PARSeq), or the head's LSE partials once per (image, position)
// and a gather per candidate (ViTSTR).
int score_impl(parseq_engine* e, const parseq_score_args* a, const void* images_any, bool u8, float* scores, float* token_lp,
               cudaStream_t user) {
  const int L = e->L, D = e->D, N = a->batch, M = a->num_candidates;
  const int bos = e->V - 2, pad = e->V - 1;
  const int ntiles = (e->C + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
  const long long img_sz = image_bytes(e, u8);
  const char* images = static_cast<const char*>(images_any);
  PQ_TRY(score_reserve(e));
  // host metadata: lengths [M], then per arch the candidates' targets / images or the groups' ids, targets, offsets
  std::vector<int> first(static_cast<size_t>(N) + 1, 0);              // first candidate of image b
  for (int b = 0; b < N; ++b) first[b + 1] = first[b] + a->per_image[b];
  std::vector<int> h(a->lengths, a->lengths + M);
  const long long len_off = 0;
  long long vt_tgt_off = 0, vt_img_off = 0;
  std::vector<ScoreGroup> groups;
  if (e->arch == 1) {
    vt_tgt_off = static_cast<long long>(h.size());
    for (int m = 0; m < M; ++m)
      for (int i = 0; i < L; ++i) h.push_back(i <= a->lengths[m] ? a->targets[1ll * m * L + i] : -1);
    vt_img_off = static_cast<long long>(h.size());
    for (int b = 0; b < N; ++b) h.insert(h.end(), static_cast<size_t>(a->per_image[b]), b);
  } else {
    const long long cap = 1ll * e->dec_chunk * L;
    std::vector<int> img_of(static_cast<size_t>(M));
    for (int b = 0; b < N; ++b) std::fill(img_of.begin() + first[b], img_of.begin() + first[b + 1], b);
    for (int b0 = 0; b0 < N; b0 += e->max_batch) {                    // groups never span super-chunks
      const int m_end = first[std::min(N, b0 + e->max_batch)];
      for (int m = first[b0]; m < m_end;) {
        ScoreGroup g{m, m, 0, img_of[m], 0, 0, 0, 0, 0};
        while (g.m1 < m_end) {
          const int P = std::max(g.P, a->lengths[g.m1] + 1);
          if (1ll * (g.m1 + 1 - g.m0) * P > cap) break;
          g.P = P;
          ++g.m1;
        }
        g.nimg = img_of[g.m1 - 1] - g.b_lo + 1;
        g.ids_off = static_cast<long long>(h.size());
        for (int c = g.m0; c < g.m1; ++c) {
          const size_t r = h.size();
          h.resize(r + e->ids_ld, pad);
          h[r] = bos;
          for (int i = 0; i < a->lengths[c]; ++i) h[r + 1 + i] = a->targets[1ll * c * L + i];
        }
        g.tgt_off = static_cast<long long>(h.size());
        for (int c = g.m0; c < g.m1; ++c)
          for (int i = 0; i < g.P; ++i) h.push_back(i <= a->lengths[c] ? a->targets[1ll * c * L + i] : -1);
        g.cand_off = static_cast<long long>(h.size());
        for (int j = 0; j <= g.nimg; ++j) {
          const int b = g.b_lo + j;
          const int c = (j == g.nimg) ? g.m1 : std::max(first[b], g.m0);
          h.push_back(c - g.m0);
          if (j > 0) g.max_rows = std::max(g.max_rows, (h.back() - h[h.size() - 2]) * g.P);
        }
        groups.push_back(g);
        m = g.m1;
      }
    }
  }
  PQ_TRY(e->sc_meta.grow(e, static_cast<long long>(h.size())));
  const int* meta = e->sc_meta;
  PQ_TRY(enter_main(e, user));
  // pageable source: the copy is staged before the call returns, so `h` may go
  PQ_CUDA(cudaMemcpyAsync(e->sc_meta, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, e->main));
  size_t gi = 0;
  for (int b0 = 0; b0 < N; b0 += e->max_batch) {
    const int Bc = std::min(N - b0, e->max_batch);
    if (e->arch == 1) {
      PQ_TRY(vitstr_chunks(e, images + b0 * img_sz, u8, Bc, [&](int o, int Bs) -> int {
        const int b = b0 + o;
        PQ_TRY(vitstr_rows(e, Bs, L, e->main));
        {
          TimedScope ts(e, e->main, CAT_SCORE, 2.0 * Bs * L * e->C * D);
          PQ_TRY(gemm_lse_launch(e->lo, e->xn, D, e->w("head.weight"), D, e->wf("head.bias"), Bs * L, e->C, D, nullptr,
                                 e->sc_vt_part, nullptr, e->main));
        }
        const int m0 = first[b], nc = first[b + Bs] - m0;
        TimedScope ts(e, e->main, CAT_SCORE, 0.0);
        return launch_k(e->lo, pq::score_reduce_kernel, dim3(static_cast<unsigned>(nc)), dim3(64), 0, e->main,
                        static_cast<const float2*>(e->sc_vt_part), ntiles, static_cast<const float*>(nullptr),
                        meta + vt_tgt_off + 1ll * m0 * L, meta + len_off, meta + vt_img_off, m0, b, L,
                        static_cast<const __nv_bfloat16*>(e->xn), e->wb("head.weight"), e->wf("head.bias"), D, scores, token_lp, L);
      }));
      continue;
    }
    PQ_TRY(encode_super(e, images + b0 * img_sz, u8, Bc));
    size_t g_end = gi;
    while (g_end < groups.size() && groups[g_end].b_lo < b0 + Bc) ++g_end;
    PQ_TRY(fan_out(e, static_cast<int>(g_end - gi), [&](int k, parseq_engine::Stage& sg, cudaStream_t ds) -> int {
      const ScoreGroup& g = groups[gi + static_cast<size_t>(k)];
      const int B = g.m1 - g.m0;
      const unsigned char* causal = e->sc_causal + 1ll * (g.P - 1) * L * L;
      DecodePass p;
      p.b_first = g.b_lo - b0; p.B = B; p.nq = g.P; p.nkeys = g.P; p.ids = meta + g.ids_off;
      p.qmask = causal; p.cmask = e->cfg.dec_depth > 1 ? causal : nullptr;
      p.cand_off = meta + g.cand_off; p.cand_imgs = g.nimg; p.cand_max_rows = g.max_rows;
      if (a->attn_maps != nullptr) {
        // the last layer's query rows of this pass, under each candidate's L map rows (0 past its EOS)
        p.maps = a->attn_maps + 1ll * g.m0 * L * e->T;
        p.maps_len = meta + len_off + g.m0;
        p.maps_ld = L;
      }
      p.tail = Tail::LogSumExp; p.lse_tgt = meta + g.tgt_off;
      PQ_TRY(decode_pass(e, sg, p, ds));
      TimedScope ts(e, ds, CAT_SCORE, 0.0);
      return launch_k(e->lo, pq::score_reduce_kernel, dim3(static_cast<unsigned>(B)), dim3(64), 0, ds,
                      static_cast<const float2*>(sg.lse_part), ntiles, static_cast<const float*>(sg.lse_tlogit),
                      static_cast<const int*>(nullptr), meta + len_off, static_cast<const int*>(nullptr), g.m0, 0, g.P,
                      static_cast<const __nv_bfloat16*>(nullptr), static_cast<const __nv_bfloat16*>(nullptr),
                      static_cast<const float*>(nullptr), D, scores, token_lp, L);
    }));
    gi = g_end;
  }
  return leave_main(e, user);
}

// Shared checks of the score entry points: the counts first (a NULL handle is enough for them), then the handle, then
// the targets against its configuration.
int check_score_call(parseq_engine* e, const parseq_score_args* a, const void* images, const float* scores) {
  PQ_TRY(check_score(a, -1, 0));
  if (images == nullptr || scores == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  if (a->attn_maps != nullptr && e->arch != 0)
    return fail(PARSEQ_ERR_UNSUPPORTED, "attn_maps: ViTSTR has no decoder cross-attention");
  return check_score(a, e->cfg.max_label_length, e->C);
}

// ---------------------------------------------------------------- beam search (parseq_beam_search)
// ViTSTR: images whose [L, C] logits one beam group holds (the head runs once per group, the selection once per position)
int beam_vt_images(const parseq_engine* e) { return std::min(e->chunk, 32); }

// Beam buffers, on the first beam call (an engine that never beam-searches allocates none of them).  PARSeq: every stage
// holds dec_chunk beam rows, whatever the beam width; ViTSTR: stage 0 holds beam_vt_images images of BEAM_MAX slots.
int beam_reserve(parseq_engine* e) {
  const size_t nst = e->arch == 0 ? e->stages.size() : 1;
  const int D = e->D;
  for (size_t s = 0; s < nst; ++s) {
    parseq_engine::Stage::Beam& bm = e->stages[s].bm;
    if (bm.rows > 0) continue;
    const int rows = e->arch == 0 ? e->dec_chunk : beam_vt_images(e) * pq::BEAM_MAX;
    const long long lrows = e->arch == 0 ? rows : 1ll * beam_vt_images(e) * e->L;
    for (int h = 0; h < 2; ++h) {
      PQ_TRY(bm.ids[h].reserve(1ll * rows * e->ids_ld, &e->beam_bytes));
      PQ_TRY(bm.score[h].reserve(rows, &e->beam_bytes));
      PQ_TRY(bm.len[h].reserve(rows, &e->beam_bytes));
      PQ_TRY(bm.st[h].reserve(rows, &e->beam_bytes));
    }
    PQ_TRY(bm.parent.reserve(rows, &e->beam_bytes));
    const long long ntiles = (e->C + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
    if (e->C <= 128) {
      PQ_TRY(bm.logits.reserve(lrows * e->C, &e->beam_bytes));
    } else {
      PQ_TRY(bm.part.reserve(lrows * ntiles, &e->beam_bytes));
      PQ_TRY(bm.keys.reserve(lrows * ntiles * pq::BEAM_TOPK_LD, &e->beam_bytes));
    }
    if (e->arch == 0 && e->cfg.dec_depth > 1) {
      bm.kvc.resize(static_cast<size_t>(e->cfg.dec_depth - 1));
      for (auto& c : bm.kvc) PQ_TRY(c.reserve(1ll * e->dec_chunk * e->L * 2 * D, &e->beam_bytes));
    }
    bm.rows = rows;
  }
  return PARSEQ_OK;
}

// ViTSTR under a lexicon: images per beam group.  Its head writes the group's [G * L, C] fp32 logits, which above 128
// classes can be large: the group holds at most 2^21 logits (8 MB; e.g. 4 images at 16384 classes and L = 26) or one image.
// At <= 128 classes this is beam_vt_images, so the plain beam's logits buffer serves.
int beam_lex_vt_images(const parseq_engine* e) {
  const long long per = 1ll * e->L * e->C;
  return static_cast<int>(std::max(1ll, std::min<long long>(beam_vt_images(e), (1ll << 21) / per)));
}

// Lexicon buffers, on the first lexicon call (after beam_reserve; counted in beam_bytes): each beam row's node,
// double-buffered, and above 128 classes the fp32 logits of a stage's rows (PARSeq: dec_chunk rows, 8 MB at 16384 classes
// and dec_chunk 128; ViTSTR: beam_lex_vt_images images' L positions).
int lexicon_reserve(parseq_engine* e) {
  const size_t nst = e->arch == 0 ? e->stages.size() : 1;
  for (size_t s = 0; s < nst; ++s) {
    parseq_engine::Stage::Beam& bm = e->stages[s].bm;
    for (int h = 0; h < 2; ++h) PQ_TRY(bm.node[h].reserve(bm.rows, &e->beam_bytes));
    const long long lrows = e->arch == 0 ? e->dec_chunk : 1ll * beam_lex_vt_images(e) * e->L;
    PQ_TRY(bm.logits.reserve(lrows * e->C, &e->beam_bytes));
  }
  return PARSEQ_OK;
}

// Beam search over a batch of images (parseq_beam_search).  PARSeq: the encoder and the cross K/V once per super-chunk as
// forward_super runs them, then groups of dec_chunk / K images (all K beams of an image in one group) round-robin over
// the stages' streams; each step is one decoder pass over the group's beam rows (decode_pass with DecodePass::beam),
// the head's logits of the step, and beam_select_kernel.  ViTSTR: the head once over a group's [B * L] token rows, then
// beam_select_kernel once per position.
int beam_impl(parseq_engine* e, const parseq_beam_args* a, const void* images_any, bool u8, int* ids, int* lengths,
              float* scores, cudaStream_t user, const parseq_lexicon* lx = nullptr, const int* roots = nullptr) {
  const int N = a->batch, K = a->beam_width, D = e->D, C = e->C, L = e->L;
  const int S = num_steps_of(e, a->max_length);
  const long long img_sz = image_bytes(e, u8);
  const char* images = static_cast<const char*>(images_any);
  PQ_TRY(beam_reserve(e));
  if (lx != nullptr) PQ_TRY(lexicon_reserve(e));
  if (a->attn_maps != nullptr) PQ_TRY(causal_reserve(e));
  auto init = [&](parseq_engine::Stage::Beam& bm, int B, cudaStream_t st) {
    const int n = B * K * e->ids_ld;
    e->launches++;
    return launch_k(e->lo, pq::beam_init_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st, bm.ids[0],
                    bm.score[0], bm.len[0], bm.st[0], B * K, K, e->ids_ld, e->V - 2, e->V - 1);
  };
  // step `step` of the group whose first image is g0 (in the call's batch)
  const bool wide = C > 128;
  const bool topk = wide && lx == nullptr;           // the head's top-K epilogue (the lexicon step reads whole rows)
  const int ntiles = (C + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N;
  if (lx != nullptr && roots != nullptr) {
    // `roots`: the checked host copy of the call's roots (beam_lexicon_call), uploaded below
    const long long cap0 = e->lex_roots.size();
    const int rc = e->lex_roots.grow(e, N);
    e->beam_bytes += 4ll * (e->lex_roots.size() - cap0);
    PQ_TRY(rc);
  }
  auto select = [&](parseq_engine::Stage::Beam& bm, int B, int step, long long row0, long long img_stride,
                    long long slot_stride, int g0, cudaStream_t st) {
    const int cur = step & 1, nxt = cur ^ 1;
    TimedScope ts(e, st, CAT_BEAM, 0.0);
    pq::BeamLex bl{};
    if (lx != nullptr)
      bl = pq::BeamLex{lx->first_edge, lx->edge_class, lx->edge_child, lx->terminal,
                       roots != nullptr ? e->lex_roots + g0 : nullptr, bm.node[cur], bm.node[nxt]};
    return launch_k(e->lo, lx != nullptr ? pq::beam_select_kernel<true> : pq::beam_select_kernel<false>,
                    dim3(static_cast<unsigned>(B)), dim3(pq::BEAM_THREADS), 0, st,
                    static_cast<const float*>(bm.logits), static_cast<const float2*>(bm.part),
                    static_cast<const unsigned long long*>(topk ? bm.keys.get() : nullptr), ntiles, row0, img_stride, slot_stride, C, K, step, S, a->class_mask ? a->class_mask + 1ll * g0 * e->mask_ld : nullptr, e->mask_ld,
                    static_cast<const int*>(bm.ids[cur]), static_cast<const float*>(bm.score[cur]),
                    static_cast<const int*>(bm.len[cur]), static_cast<const int*>(bm.st[cur]), bm.ids[nxt], bm.score[nxt],
                    bm.len[nxt], bm.st[nxt], bm.parent, e->ids_ld, ids + 1ll * g0 * K * S, lengths + 1ll * g0 * K,
                    scores + 1ll * g0 * K, bl);
  };
  PQ_TRY(enter_main(e, user));
  // pageable source (a std::vector of beam_lexicon_call): the copy is staged before the call returns
  if (lx != nullptr && roots != nullptr)
    PQ_CUDA(cudaMemcpyAsync(e->lex_roots, roots, 4ull * N, cudaMemcpyHostToDevice, e->main));
  for (int b0 = 0; b0 < N; b0 += e->max_batch) {
    const int Bc = std::min(N - b0, e->max_batch);
    if (e->arch == 1) {
      parseq_engine::Stage::Beam& bm = e->stages[0].bm;
      const int G = lx != nullptr ? beam_lex_vt_images(e) : beam_vt_images(e);
      PQ_TRY(vitstr_chunks(e, images + b0 * img_sz, u8, Bc, [&](int o, int Bs) -> int {
        PQ_TRY(vitstr_rows(e, Bs, L, e->main));
        for (int g = 0; g < Bs; g += G) {
          const int Bg = std::min(G, Bs - g);
          if (topk) {
            // the top-K epilogue over the group's [Bg * L] token rows: row r belongs to image r / L
            TimedScope ts(e, e->main, CAT_DEC_GEMM, 2.0 * Bg * L * C * D);
            PQ_TRY(gemm_topk_launch(e->lo, e->xn + 1ll * g * L * D, D, e->w("head.weight"), D, e->wf("head.bias"), Bg * L, C, D, K,
                                    a->class_mask ? a->class_mask + 1ll * (b0 + o + g) * e->mask_ld : nullptr, L, bm.part,
                                    bm.keys, e->main));
          } else {
            PQ_TRY(gemm(e, e->xn + 1ll * g * L * D, D, e->w("head.weight"), D, e->wf("head.bias"), Bg * L, C, D, pq::EPI_F32,
                        1.0f, nullptr, 0, 0, bm.logits, C, e->main));
          }
          PQ_TRY(init(bm, Bg, e->main));
          for (int step = 0; step < S; ++step) PQ_TRY(select(bm, Bg, step, step, L, 0, b0 + o + g, e->main));
        }
        return PARSEQ_OK;
      }));
      continue;
    }
    PQ_TRY(encode_super(e, images + b0 * img_sz, u8, Bc));
    const int G = e->dec_chunk / K;                    // images per group: G * K beam rows fill a stage's buffers
    PQ_TRY(fan_out(e, (Bc + G - 1) / G, [&](int gi, parseq_engine::Stage& sg, cudaStream_t ds) -> int {
      parseq_engine::Stage::Beam& bm = sg.bm;
      const int g0 = gi * G, Bg = std::min(G, Bc - g0), R = Bg * K;
      PQ_TRY(init(bm, Bg, ds));
      DecodePass p;
      p.b_first = g0; p.B = R; p.nq = 1; p.ar_step = true; p.beam = K;
      if (topk) {
        p.tail = Tail::TopK; p.part = bm.part; p.keys = bm.keys; p.k = K;
        p.mask = a->class_mask ? a->class_mask + 1ll * (b0 + g0) * e->mask_ld : nullptr;
      } else {
        p.logits = bm.logits; p.logits_ld = C;
      }
      const std::vector<__nv_bfloat16*> kvc0(sg.kvc.begin(), sg.kvc.end());
      int rc = PARSEQ_OK;
      for (int step = 0; step < S && rc == PARSEQ_OK; ++step) {
        // query position `step` over keys 0..step of every beam row; the head leaves row r's logits at bm.logits + r * C
        // (<= 128 classes, and at every C under a lexicon: the chain's head GEMM, no argmax) or its partials and top-K
        // keys (above)
        p.q0 = step; p.nkeys = step + 1; p.ids = bm.ids[step & 1];
        rc = decode_pass(e, sg, p, ds);
        if (rc == PARSEQ_OK) rc = select(bm, Bg, step, 0, K, 1, b0 + g0, ds);
        if (rc != PARSEQ_OK || e->cfg.dec_depth == 1 || step + 1 == S) continue;
        // depth >= 2: each new beam row continues its parent's content K/V cache rows 0..step
        TimedScope ts(e, ds, CAT_BEAM, 0.0);
        const long long pitch4 = 1ll * L * 2 * D * 2 / 16;
        const int n4 = (step + 1) * 2 * D * 2 / 16;
        for (size_t l = 0; l < sg.kvc.size() && rc == PARSEQ_OK; ++l) {
          const long long total = 1ll * R * n4;
          rc = launch_k(e->lo, pq::beam_kv_gather_kernel, dim3(static_cast<unsigned>(std::min<long long>((total + 255) / 256, 132ll * 8))),
                        dim3(256), 0, ds, reinterpret_cast<const uint4*>(sg.kvc[l].get()), reinterpret_cast<uint4*>(bm.kvc[l].get()),
                        static_cast<const int*>(bm.parent), R, pitch4, n4);
          std::swap(sg.kvc[l], bm.kvc[l]);
        }
      }
      // the stage's own cache pointers back (their contents are scratch between calls)
      for (size_t l = 0; l < sg.kvc.size(); ++l)
        if (sg.kvc[l] != kvc0[l]) std::swap(sg.kvc[l], bm.kvc[l]);
      if (rc != PARSEQ_OK || a->attn_maps == nullptr) return rc;
      // the final hypotheses' maps: the last selection left each row's [BOS, c_1..] in bm.ids[S & 1] (valid ids
      // everywhere), so one teacher-forced pass over the rows' first S ids under the causal masks computes every step's
      // query; image j's K * S query rows are contiguous
      float* const maps = a->attn_maps + 1ll * (b0 + g0) * K * S * e->T;
      PQ_TRY(ar_maps_pass(e, sg, g0, R, S, bm.ids[S & 1], maps, ds, K));
      TimedScope ts(e, ds, CAT_MAPS, 0.0);
      return launch_k(e->lo, pq::maps_zero_tail_kernel, dim3(static_cast<unsigned>(R)), dim3(256), 0, ds, maps,
                      static_cast<const int*>(lengths + 1ll * (b0 + g0) * K), S, e->T);
    }));
  }
  return leave_main(e, user);
}

// The host checks of a lexicon (parseq_lexicon_check) against C head classes and labels of at most max_label_length
int check_lexicon(const parseq_lexicon_desc* d, int num_classes, int max_label_length) {
  if (d == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  const int V = d->num_nodes, E = d->num_edges;
  if (V <= 0 || E < 0) return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: num_nodes must be >= 1 and num_edges >= 0");
  if (d->first_edge == nullptr || d->terminal == nullptr || (E > 0 && (d->edge_class == nullptr || d->edge_child == nullptr)))
    return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: null array");
  if (d->first_edge[0] != 0 || d->first_edge[V] != E)
    return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: first_edge must start at 0 and end at num_edges = " + std::to_string(E));
  std::vector<int> depth(static_cast<size_t>(V), 0);   // longest path ending at each node, in index order
  for (int v = 0; v < V; ++v) {
    const int e0 = d->first_edge[v], e1 = d->first_edge[v + 1];
    if (e1 < e0 || e1 > E) return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: first_edge is not monotone at node " + std::to_string(v));
    for (int j = e0; j < e1; ++j) {
      const int c = d->edge_class[j], ch = d->edge_child[j];
      if (c < 1 || c >= num_classes)
        return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: edge " + std::to_string(j) + " has class " + std::to_string(c) +
                                                ", outside 1.." + std::to_string(num_classes - 1));
      if (j > e0 && c <= d->edge_class[j - 1])
        return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: edge classes of node " + std::to_string(v) +
                                                " are not strictly increasing");
      if (ch <= v || ch >= V)
        return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: edge " + std::to_string(j) + " of node " + std::to_string(v) +
                                                " has child " + std::to_string(ch) + ", not in " + std::to_string(v + 1) +
                                                ".." + std::to_string(V - 1));
      depth[static_cast<size_t>(ch)] = std::max(depth[static_cast<size_t>(ch)], depth[static_cast<size_t>(v)] + 1);
    }
    if (depth[static_cast<size_t>(v)] > max_label_length)
      return fail(PARSEQ_ERR_INVALID_ARG, "lexicon: a path of " + std::to_string(depth[static_cast<size_t>(v)]) +
                                              " characters, more than max_label_length = " + std::to_string(max_label_length));
  }
  return PARSEQ_OK;
}

// Checks of the beam entry points, all on the host before anything is launched.
int check_beam_call(parseq_engine* e, const parseq_beam_args* a, const void* images, const int* ids, const int* lengths,
                    const float* scores) {
  if (a == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (a->batch < 0) return fail(PARSEQ_ERR_INVALID_ARG, "negative batch");
  if (a->beam_width < 1 || a->beam_width > pq::BEAM_MAX)
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_width " + std::to_string(a->beam_width) + " outside [1, 16]");
  if (a->max_length < -1) return fail(PARSEQ_ERR_INVALID_ARG, "max_length must be -1 (None) or >= 0");
  if (a->batch > 0 && (images == nullptr || ids == nullptr || lengths == nullptr || scores == nullptr))
    return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  if (a->attn_maps != nullptr && e->arch != 0)
    return fail(PARSEQ_ERR_UNSUPPORTED, "attn_maps: ViTSTR has no decoder cross-attention");
  if (e->arch == 0 && a->beam_width > e->dec_chunk)
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_width " + std::to_string(a->beam_width) + " exceeds the decoder chunk (option "
                                        "dec_chunk = " + std::to_string(e->dec_chunk) + ")");
  return PARSEQ_OK;
}

// The lexicon beam entry points: the beam checks, the lexicon against the engine, every root a node; then beam_impl
int beam_lexicon_call(parseq_engine* e, const parseq_beam_args* a, const parseq_lexicon* lx, const int32_t* roots,
                      const void* images, bool u8, int32_t* ids, int32_t* lengths, float* scores, parseq_stream_t stream) {
  PQ_TRY(check_beam_call(e, a, images, ids, lengths, scores));
  if (lx == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null lexicon");
  if (lx->device != e->cfg.device || lx->C != e->C)
    return fail(PARSEQ_ERR_INVALID_ARG, "lexicon was made for device " + std::to_string(lx->device) + " and " +
                                            std::to_string(lx->C) + " classes, the engine has device " +
                                            std::to_string(e->cfg.device) + " and " + std::to_string(e->C));
  // the roots are read once, into a host copy that is checked and then uploaded: the caller's buffer (pageable or
  // pinned) may change as soon as the call returns, and the device only ever sees checked values
  std::vector<int> rv;
  if (roots != nullptr) {
    rv.assign(roots, roots + a->batch);
    for (int b = 0; b < a->batch; ++b)
      if (rv[static_cast<size_t>(b)] < 0 || rv[static_cast<size_t>(b)] >= lx->V)
        return fail(PARSEQ_ERR_INVALID_ARG, "root " + std::to_string(rv[static_cast<size_t>(b)]) + " of image " +
                                                std::to_string(b) + " is not a node of the lexicon (0.." +
                                                std::to_string(lx->V - 1) + ")");
  }
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  return beam_impl(e, a, images, u8, ids, lengths, scores, reinterpret_cast<cudaStream_t>(stream), lx,
                   roots != nullptr ? rv.data() : nullptr);
}

}  // namespace

// =============================================================================== C ABI
extern "C" {

const char* parseq_last_error(void) { return g_last_error.c_str(); }
const char* parseq_version(void) { return "parseq_b200 0.2 (sm_90a, wgmma/TMA)"; }

int parseq_create(const parseq_config* cfg, parseq_engine** out) {
  if (cfg == nullptr || out == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(PARSEQ_ERR_NO_DEVICE, "no CUDA device: parseq_b200 has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(PARSEQ_ERR_INVALID_ARG, "bad device ordinal");
  PQ_CUDA(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  PQ_CUDA(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(PARSEQ_ERR_NO_DEVICE, std::string("device is sm_") + std::to_string(prop.major * 10 + prop.minor) +
                                          ", the kernels are sm_90a (H100) only");
  const int sm_count = prop.multiProcessorCount;
  PQ_TRY(ensure_kernel_attributes());
  PQ_TRY(load_driver_api());
  if (cfg->arch != 0 && cfg->arch != 1) return fail(PARSEQ_ERR_INVALID_ARG, "arch: 0 (PARSeq) or 1 (ViTSTR)");
  const bool vitstr = cfg->arch == 1;
  if (!vitstr && cfg->dec_depth < 1) return fail(PARSEQ_ERR_UNSUPPORTED, "dec_depth must be >= 1 (decoder layers)");
  if (cfg->img_h % cfg->patch_h || cfg->img_w % cfg->patch_w) return fail(PARSEQ_ERR_INVALID_ARG, "img/patch mismatch");
  const int D = cfg->embed_dim;
  if (D != 192 && D != 384 && D != 768) return fail(PARSEQ_ERR_UNSUPPORTED, "embed_dim must be 192, 384 or 768");
  if (D != cfg->enc_num_heads * 64) return fail(PARSEQ_ERR_UNSUPPORTED, "encoder head_dim must be 64");
  if (!vitstr && D != cfg->dec_num_heads * 32) return fail(PARSEQ_ERR_UNSUPPORTED, "decoder head_dim must be 32");
  // L = max_label_length + 1 <= 64 decode positions: the decoder's id rows are 32 or 64 wide (DESIGN.md section 4)
  if (cfg->max_label_length > kMaxLabelLength)
    return fail(PARSEQ_ERR_UNSUPPORTED, "max_label_length must be <= 63 (labels of at most 63 characters)");
  if (cfg->max_label_length < 0) return fail(PARSEQ_ERR_INVALID_ARG, "negative max_label_length");
  // at most 16384 head classes (charset_train of <= 16383 characters): every index into the (position, token) K/V table
  // [L * V, 2D] stays in int32 (64 * 16386 * 1536 < 2^31); the table is at most 3.2 GB (DESIGN.md section 4)
  if (cfg->num_tokens < 4 || cfg->num_tokens - 2 > kMaxHeadClasses)
    return fail(PARSEQ_ERR_UNSUPPORTED, "num_tokens must be in [4, 16386] (at most 16384 head classes, charset_train of "
                                        "at most 16383 characters)");
  if (cfg->enc_mlp_ratio < 1 || cfg->enc_depth < 1) return fail(PARSEQ_ERR_INVALID_ARG, "enc_mlp_ratio / enc_depth");
  // decoder MLP: 128-wide linear1 tiles and a 3-way split-K of linear2 in 64-element k-blocks
  if (!vitstr && (cfg->dec_mlp_ratio < 1 || (D * cfg->dec_mlp_ratio) % 384 != 0))
    return fail(PARSEQ_ERR_UNSUPPORTED, "embed_dim * dec_mlp_ratio must be a multiple of 384");
  auto* e = new parseq_engine();
  e->cfg = *cfg;
  e->lo = g_default_opts;         // process defaults (parseq_set_option(NULL, ...)) seed a new handle
  e->lo.sm_count = sm_count;
  if (vitstr) {                     // no decoder: neutral values keep the (unused) decoder workspace sizes sane
    e->cfg.dec_num_heads = D / 32;
    e->cfg.dec_mlp_ratio = 1;
    e->cfg.dec_depth = 0;
  }
  cfg = &e->cfg;
  e->arch = cfg->arch;
  e->D = D;
  e->gh = cfg->img_h / cfg->patch_h;
  e->gw = cfg->img_w / cfg->patch_w;
  e->Tp = e->gh * e->gw;
  e->T = e->Tp + (vitstr ? 1 : 0);   // class token (timm VisionTransformer default, kept by vitstr/model.py)
  e->Kp = 3 * cfg->patch_h * cfg->patch_w;
  e->Me = D * cfg->enc_mlp_ratio;
  e->Md = D * cfg->dec_mlp_ratio;
  e->L = cfg->max_label_length + 1;
  e->ids_ld = e->L <= 32 ? 32 : 64;
  e->V = cfg->num_tokens;
  e->C = cfg->num_tokens - 2;
  e->mask_ld = (e->C + 31) / 32;
  e->dh_dec = D / cfg->dec_num_heads;
  e->max_batch = cfg->max_batch > 0 ? cfg->max_batch : 512;
  // One pipeline stage per super-chunk by default: the decoder chain is latency-bound and the encoder GEMMs occupy
  // every SM, so splitting into stages only shrinks the GEMMs ("chunk" option re-enables it).
  e->chunk = e->max_batch;
  e->dec_chunk = e->max_batch < 128 ? e->max_batch : 128;
  if (e->T > 256) {
    delete e;
    return fail(PARSEQ_ERR_UNSUPPORTED, "at most 256 image tokens (img_size / patch_size) are supported");
  }
  if (vitstr && e->Tp < e->L) {     // vitstr/model.py:21 slices max_length + 2 tokens out of the T + 1 available
    delete e;
    return fail(PARSEQ_ERR_UNSUPPORTED, "ViTSTR needs at least max_label_length + 1 patches");
  }
  if ((e->Kp * 2) % 16 != 0) { delete e; return fail(PARSEQ_ERR_UNSUPPORTED, "patch dim must be a multiple of 8"); }
  // ---- weight slots: state_dict keys of strhub.models.parseq.model.PARSeq ----
  // ---- (arch 1: keys of vitstr.model.ViTSTR = timm VisionTransformer; the public names drop "encoder.") ----
  if (vitstr) add_slot(e, "encoder.cls_token", D, false);
  add_slot(e, "encoder.pos_embed", 1ll * e->T * D, false);
  add_slot(e, "encoder.patch_embed.proj.weight", 1ll * D * e->Kp, true);
  add_slot(e, "encoder.patch_embed.proj.bias", D, false);
  for (int i = 0; i < cfg->enc_depth; ++i) {
    const std::string p = "encoder.blocks." + std::to_string(i) + ".";
    add_slot(e, p + "norm1.weight", D, false);
    add_slot(e, p + "norm1.bias", D, false);
    add_slot(e, p + "attn.qkv.weight", 3ll * D * D, true);
    add_slot(e, p + "attn.qkv.bias", 3 * D, false);
    add_slot(e, p + "attn.proj.weight", 1ll * D * D, true);
    add_slot(e, p + "attn.proj.bias", D, false);
    add_slot(e, p + "norm2.weight", D, false);
    add_slot(e, p + "norm2.bias", D, false);
    add_slot(e, p + "mlp.fc1.weight", 1ll * e->Me * D, true);
    add_slot(e, p + "mlp.fc1.bias", e->Me, false);
    add_slot(e, p + "mlp.fc2.weight", 1ll * D * e->Me, true);
    add_slot(e, p + "mlp.fc2.bias", D, false);
  }
  add_slot(e, "encoder.norm.weight", D, false);
  add_slot(e, "encoder.norm.bias", D, false);
  for (int l = 0; !vitstr && l < cfg->dec_depth; ++l) {
    const std::string Ly = "decoder.layers." + std::to_string(l) + ".";
    for (const char* att : {"self_attn", "cross_attn"}) {
      add_slot(e, Ly + att + ".in_proj_weight", 3ll * D * D, true);
      add_slot(e, Ly + att + ".in_proj_bias", 3 * D, false);
      add_slot(e, Ly + att + ".out_proj.weight", 1ll * D * D, true);
      add_slot(e, Ly + att + ".out_proj.bias", D, false);
    }
    add_slot(e, Ly + "linear1.weight", 1ll * e->Md * D, true);
    add_slot(e, Ly + "linear1.bias", e->Md, false);
    add_slot(e, Ly + "linear2.weight", 1ll * D * e->Md, true);
    add_slot(e, Ly + "linear2.bias", D, false);
    for (const char* n : {"norm1", "norm2", "norm_q", "norm_c"}) {
      add_slot(e, Ly + n + ".weight", D, false);
      add_slot(e, Ly + n + ".bias", D, false);
    }
  }
  if (!vitstr) {
    add_slot(e, "decoder.norm.weight", D, false);
    add_slot(e, "decoder.norm.bias", D, false);
  }
  add_slot(e, "head.weight", 1ll * e->C * D, true);
  add_slot(e, "head.bias", e->C, false);
  if (!vitstr) {
    add_slot(e, "text_embed.embedding.weight", 1ll * e->V * D, false);
    add_slot(e, "pos_queries", 1ll * e->L * D, false);
  }
  for (auto& s : e->slots) {
    // +64 elements of slack: head.bias (95 floats) is read with float4 only when in range, but keep
    // every buffer 16-byte padded
    const size_t bytes = static_cast<size_t>(s.numel + 64) * (s.bf16 ? 2 : 4);
    if (s.dev.alloc(static_cast<long long>(bytes)) != PARSEQ_OK) { parseq_destroy(e); return fail(PARSEQ_ERR_CUDA, "cudaMalloc weights"); }
    cudaMemset(s.dev, 0, bytes);
  }
  int r = e->kvtab.alloc(1ll * e->L * e->V * 2 * D);
  if (r == PARSEQ_OK) r = e->qs.alloc(1ll * e->L * D);
  if (r == PARSEQ_OK) r = alloc_workspace(e);
  if (r == PARSEQ_OK) r = make_stream(&e->main);
  if (r == PARSEQ_OK) r = make_stream(&e->copy);
  for (Event* ev : {&e->ev_c[0], &e->ev_c[1], &e->ev_c[2], &e->ev_in, &e->ev_out})
    if (r == PARSEQ_OK) r = make_event(ev);
  if (r != PARSEQ_OK) { parseq_destroy(e); return r; }
  *out = e;
  return PARSEQ_OK;
}

void parseq_destroy(parseq_engine* e) {
  if (e == nullptr) return;
  cudaSetDevice(e->cfg.device);
  cudaDeviceSynchronize();
  delete e;
}

int parseq_num_weights(const parseq_engine* e) { return e ? static_cast<int>(e->slots.size()) : 0; }
const char* parseq_weight_key(const parseq_engine* e, int i, int64_t* numel) {
  if (e == nullptr || i < 0 || i >= static_cast<int>(e->slots.size())) return nullptr;
  if (numel) *numel = e->slots[i].numel;
  return e->slots[i].pub.c_str();
}

int parseq_set_weight(parseq_engine* e, const char* key, const float* data, int64_t numel) {
  if (e == nullptr || key == nullptr || data == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  auto it = e->pub_index.find(key);
  if (it == e->pub_index.end()) return fail(PARSEQ_ERR_INVALID_ARG, std::string("unexpected state_dict key: ") + key);
  Slot& s = e->slots[it->second];
  if (numel != s.numel)
    return fail(PARSEQ_ERR_INVALID_ARG, std::string("size mismatch for ") + key + ": got " + std::to_string(numel) +
                                            ", expected " + std::to_string(s.numel));
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  if (s.bf16) {
    std::vector<uint16_t> tmp(static_cast<size_t>(numel));
    for (int64_t i = 0; i < numel; ++i) tmp[static_cast<size_t>(i)] = f32_to_bf16_rne(data[i]);
    PQ_CUDA(cudaMemcpy(s.dev, tmp.data(), tmp.size() * 2, cudaMemcpyHostToDevice));
  } else {
    PQ_CUDA(cudaMemcpy(s.dev, data, static_cast<size_t>(numel) * 4, cudaMemcpyHostToDevice));
  }
  s.set = true;
  e->finalized = false;
  return PARSEQ_OK;
}

int parseq_finalize(parseq_engine* e, parseq_stream_t stream) {
  if (e == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null engine");
  for (auto& s : e->slots)
    if (!s.set) return fail(PARSEQ_ERR_STATE, "weight not set: " + s.pub);
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  if (e->arch == 1) {               // ViTSTR has no input-independent tables
    e->finalized = true;
    return PARSEQ_OK;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int D = e->D, L = e->L, V = e->V;
  const std::string Ly = "decoder.layers.0.";
  const long long rows = 1ll * L * V;
  DevBuf<float> ctx;                // temporaries, freed on return (after the synchronise below)
  DevBuf<__nv_bfloat16> ctxn, qn;
  PQ_TRY(ctx.alloc(rows * D));
  PQ_TRY(ctxn.alloc(rows * D));
  PQ_TRY(qn.alloc(1ll * L * D));
  int r = PARSEQ_OK;
  pq::build_ctx_rows_kernel<<<1024, 256, 0, st>>>(e->wf("text_embed.embedding.weight"), e->wf("pos_queries"), ctx, L, V, D,
                                                  std::sqrt(static_cast<float>(D)));
  if (cudaGetLastError() != cudaSuccess) r = fail(PARSEQ_ERR_CUDA, "build_ctx_rows_kernel launch");
  if (r == PARSEQ_OK) r = layernorm_launch(e->lo, ctx, e->wf(Ly + "norm_c.weight"), e->wf(Ly + "norm_c.bias"), 1e-5f, static_cast<int>(rows), D,
                           ctxn, nullptr, st);
  // content K/V for every (position, token): rows D..3D-1 of self_attn.in_proj (enc-dec packed projection)
  if (r == PARSEQ_OK)
    r = gemm_launch(e->lo, ctxn, D, e->wb(Ly + "self_attn.in_proj_weight") + 1ll * D * D, D,
                    e->wf(Ly + "self_attn.in_proj_bias") + D, static_cast<int>(rows), 2 * D, D, pq::EPI_BF16, 1.0f, nullptr,
                    0, 0, e->kvtab, 2 * D, st);
  // query projections of the (input independent) position queries, pre-scaled by 1/sqrt(head_dim)
  if (r == PARSEQ_OK)
    r = layernorm_launch(e->lo, e->wf("pos_queries"), e->wf(Ly + "norm_q.weight"), e->wf(Ly + "norm_q.bias"), 1e-5f, L, D, qn,
                         nullptr, st);
  if (r == PARSEQ_OK)
    r = gemm_launch(e->lo, qn, D, e->wb(Ly + "self_attn.in_proj_weight"), D, e->wf(Ly + "self_attn.in_proj_bias"), L, D, D,
                    pq::EPI_F32, 1.0f / std::sqrt(static_cast<float>(e->dh_dec)), nullptr, 0, 0, e->qs, D, st);
  cudaError_t ce = cudaStreamSynchronize(st);
  if (r != PARSEQ_OK) return r;
  if (ce != cudaSuccess) return fail(PARSEQ_ERR_CUDA, std::string("finalize: ") + cudaGetErrorString(ce));
  e->ar2_maps_ok = false;
  if (ar_path(e) == ArPath::Cluster) PQ_TRY(ar2_build_maps(e));
  e->finalized = true;
  return PARSEQ_OK;
}

int parseq_forward(parseq_engine* e, const parseq_forward_args* a, const float* images, float* logits, int32_t* ids,
                   int32_t* steps, parseq_stream_t stream) {
  return forward_call(e, a, images, logits, ids, steps, stream, false, false);
}

int parseq_forward_host(parseq_engine* e, const parseq_forward_args* a, const float* images_host, float* logits_host,
                        int32_t* ids_host, int32_t* steps_host, parseq_stream_t stream) {
  return forward_call(e, a, images_host, logits_host, ids_host, steps_host, stream, true, false);
}

int parseq_forward_u8(parseq_engine* e, const parseq_forward_args* a, const uint8_t* images_hwc, float* logits, int32_t* ids,
                      int32_t* steps, parseq_stream_t stream) {
  return forward_call(e, a, images_hwc, logits, ids, steps, stream, false, true);
}

int parseq_forward_host_u8(parseq_engine* e, const parseq_forward_args* a, const uint8_t* images_hwc_host, float* logits_host,
                           int32_t* ids_host, int32_t* steps_host, parseq_stream_t stream) {
  return forward_call(e, a, images_hwc_host, logits_host, ids_host, steps_host, stream, true, true);
}

int parseq_resize_crops(parseq_engine* e, int32_t batch, const parseq_crops* crops, uint8_t* out_hwc, parseq_stream_t stream) {
  if (batch < 0) return fail(PARSEQ_ERR_INVALID_ARG, "negative batch");
  PQ_TRY(check_crops(batch, crops));
  if (out_hwc == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e, false));
  PQ_TRY(check_crop_smem(e, batch, crops));
  if (batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  const CropBatch cb{crops, false};
  PQ_TRY(enter_main(e, user));
  for (int b0 = 0; b0 < batch; b0 += e->max_batch) {
    const int Bc = (batch - b0 < e->max_batch) ? (batch - b0) : e->max_batch;
    PQ_TRY(crops_table(e, cb, b0, Bc, e->main));
    PQ_TRY(crops_resize(e, cb, b0, 0, Bc, out_hwc + 3ll * e->cfg.img_h * e->cfg.img_w * b0, e->main));
  }
  return leave_main(e, user);
}

int parseq_warp_regions(parseq_engine* e, int32_t count, const parseq_regions* r, uint8_t* out, int64_t out_bytes,
                        parseq_stream_t stream) {
  long long packed = 0;
  PQ_TRY(check_regions(count, r, out, out_bytes, &packed));
  PQ_TRY(check_ready(e, false));
  if (count == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  PQ_TRY(e->reg_tab.grow(e, e->max_batch));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  PQ_TRY(enter_main(e, user));
  long long dst = 0;
  for (int b0 = 0; b0 < count; b0 += e->max_batch) {
    const int Bc = (count - b0 < e->max_batch) ? (count - b0) : e->max_batch;
    e->reg_descs.resize(static_cast<size_t>(Bc));
    long long pixels = 0;                  // of the largest region of the chunk: the grid's tile count
    for (int i = 0; i < Bc; ++i) {
      const int g = b0 + i, f = r->frame_index[g];
      pq::RegionDesc& d = e->reg_descs[static_cast<size_t>(i)];
      std::memcpy(d.a, r->coeffs + 8ll * g, sizeof(d.a));
      d.src = r->frame_offsets[f];
      d.dst = dst;
      d.fh = r->frame_sizes[2 * f];
      d.fw = r->frame_sizes[2 * f + 1];
      d.h = r->sizes[2 * g];
      d.w = r->sizes[2 * g + 1];
      dst += 3ll * d.h * d.w;
      pixels = std::max(pixels, 1ll * d.h * d.w);
    }
    // pageable source: the copy is staged when it returns, so reg_descs may change for the next chunk
    PQ_CUDA(cudaMemcpyAsync(e->reg_tab, e->reg_descs.data(), sizeof(pq::RegionDesc) * Bc, cudaMemcpyHostToDevice, e->main));
    const dim3 grid(static_cast<unsigned>((pixels + pq::REGION_THREADS - 1) / pq::REGION_THREADS), static_cast<unsigned>(Bc));
    TimedScope ts(e, e->main, CAT_MISC, 0.0);
    // no PDL: the kernel reads the table copy and the caller's frames
    PQ_TRY(launch_ex(LaunchConfig(grid, dim3(pq::REGION_THREADS), 0, e->main, 0, false), pq::region_warp_kernel,
                     r->frames, static_cast<const pq::RegionDesc*>(e->reg_tab), out));
  }
  return leave_main(e, user);
}

int parseq_tps_coeffs(int32_t num_points, const double* points, double* coeffs) {
  if (points == nullptr || coeffs == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null points or coeffs");
  PQ_TRY(check_polygon_points("", num_points, points));
  tps_solve(num_points / 2, points, coeffs);
  return PARSEQ_OK;
}

int parseq_warp_polygons(parseq_engine* e, int32_t count, const parseq_polygons* r, uint8_t* out, int64_t out_bytes,
                         parseq_stream_t stream) {
  long long packed = 0;
  PQ_TRY(check_polygons(count, r, out, out_bytes, &packed));
  PQ_TRY(check_ready(e, false));
  if (count == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  PQ_TRY(e->tps_tab.grow(e, e->max_batch));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  PQ_TRY(enter_main(e, user));
  long long dst = 0, first = 0;
  for (int b0 = 0; b0 < count; b0 += e->max_batch) {
    const int Bc = (count - b0 < e->max_batch) ? (count - b0) : e->max_batch;
    e->tps_descs.resize(static_cast<size_t>(Bc));
    long long pixels = 0;                  // of the largest region of the chunk: the grid's tile count
    for (int i = 0; i < Bc; ++i) {
      const int g = b0 + i, f = r->frame_index[g];
      pq::TpsDesc& d = e->tps_descs[static_cast<size_t>(i)];
      std::memset(&d, 0, sizeof(d));
      d.k = r->num_points[g] / 2;
      tps_solve(d.k, r->points + 2 * first, d.t);
      tps_cx(d.k, d.cx);
      first += r->num_points[g];
      d.src = r->frame_offsets[f];
      d.dst = dst;
      d.fh = r->frame_sizes[2 * f];
      d.fw = r->frame_sizes[2 * f + 1];
      d.h = r->sizes[2 * g];
      d.w = r->sizes[2 * g + 1];
      dst += 3ll * d.h * d.w;
      pixels = std::max(pixels, 1ll * d.h * d.w);
    }
    // pageable source: the copy is staged when it returns, so tps_descs may change for the next chunk
    PQ_CUDA(cudaMemcpyAsync(e->tps_tab, e->tps_descs.data(), sizeof(pq::TpsDesc) * Bc, cudaMemcpyHostToDevice, e->main));
    const dim3 grid(static_cast<unsigned>((pixels + pq::REGION_THREADS - 1) / pq::REGION_THREADS), static_cast<unsigned>(Bc));
    TimedScope ts(e, e->main, CAT_MISC, 0.0);
    // no PDL: the kernel reads the table copy and the caller's frames
    PQ_TRY(launch_ex(LaunchConfig(grid, dim3(pq::REGION_THREADS), 0, e->main, 0, false), pq::region_tps_kernel,
                     r->frames, static_cast<const pq::TpsDesc*>(e->tps_tab), out));
  }
  return leave_main(e, user);
}

int parseq_forward_crops(parseq_engine* e, const parseq_forward_args* a, const parseq_crops* crops, float* logits, int32_t* ids,
                         int32_t* steps, parseq_stream_t stream) {
  PQ_TRY(check_crops_call(e, a, crops, logits));
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  const CropBatch cb{crops, false};
  return forward_impl(e, a, nullptr, logits, ids, steps, reinterpret_cast<cudaStream_t>(stream), false, true, &cb);
}

int parseq_forward_host_crops(parseq_engine* e, const parseq_forward_args* a, const parseq_crops* crops, float* logits_host,
                              int32_t* ids_host, int32_t* steps_host, parseq_stream_t stream) {
  PQ_TRY(check_crops_call(e, a, crops, logits_host));
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  const CropBatch cb{crops, true};
  PQ_TRY(crops_reserve(e, cb, a->batch));
  PQ_TRY(forward_impl(e, a, nullptr, logits_host, ids_host, steps_host, reinterpret_cast<cudaStream_t>(stream), true, true, &cb));
  PQ_CUDA(cudaStreamSynchronize(e->main));
  return PARSEQ_OK;
}

int parseq_forward_crops_oriented(parseq_engine* e, const parseq_forward_args* a, const parseq_crops* crops,
                                  const parseq_orient_args* o, float* logits, int32_t* ids, int32_t* steps,
                                  parseq_stream_t stream) {
  PQ_TRY(check_orient(o));
  if (crops == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (crops->rotations != nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "rotations must be NULL: the oriented call chooses each crop's rotation");
  parseq_crops c = *crops;
  c.rotation = o->orientations[0];
  PQ_TRY(check_crops_call(e, a, &c, logits));
  const int R = o->num_orientations;
  if (e->max_batch < R - 1)
    return fail(PARSEQ_ERR_INVALID_ARG, "max_batch (" + std::to_string(e->max_batch) + ") must be >= num_orientations - 1 (" +
                                            std::to_string(R - 1) + "): a crop's readings share one super-chunk");
  if (a->attn_maps != nullptr && e->arch != 0)
    return fail(PARSEQ_ERR_UNSUPPORTED, "attn_maps: ViTSTR has no decoder cross-attention");
  for (int r = 1; r < R; ++r) {
    parseq_crops cr = c;
    cr.rotation = o->orientations[r];
    PQ_TRY(check_crop_smem(e, a->batch, &cr));
  }
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  const cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  cudaPointerAttributes pa{};
  const bool on_device = cudaPointerGetAttributes(&pa, c.data) == cudaSuccess &&
                         (pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged);
  cudaGetLastError();
  if (!on_device) {
    // host crops: the staging buffer holds one super-chunk's bytes at a time - pass 1's span of max_batch crops, or the
    // listed crops of a pass-2 super-chunk, at most the floor(max_batch / (R - 1)) largest crops
    const CropBatch cb{&c, true};
    PQ_TRY(crops_reserve(e, cb, a->batch));
    if (R > 1) {
      std::vector<long long> bytes(static_cast<size_t>(a->batch));
      for (int i = 0; i < a->batch; ++i) bytes[static_cast<size_t>(i)] = 3ll * c.sizes[2 * i] * c.sizes[2 * i + 1];
      const size_t per = std::min(bytes.size(), static_cast<size_t>(e->max_batch / (R - 1)));
      std::partial_sort(bytes.begin(), bytes.begin() + static_cast<long>(per), bytes.end(), std::greater<long long>());
      long long need = 0;
      for (size_t i = 0; i < per; ++i) need += bytes[i];
      PQ_TRY(e->crop_stage.grow(e, need));
    }
  }
  return orient_impl(e, a, c, !on_device, o, logits, ids, steps, user);
}

int parseq_score_check(const parseq_config* cfg, const parseq_score_args* a) {
  if (cfg == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (a != nullptr && a->attn_maps != nullptr && cfg->arch != 0)
    return fail(PARSEQ_ERR_UNSUPPORTED, "attn_maps: ViTSTR has no decoder cross-attention");
  return check_score(a, cfg->max_label_length, cfg->num_tokens - 2);
}

int parseq_score(parseq_engine* e, const parseq_score_args* a, const float* images, float* scores, float* token_logprobs,
                 parseq_stream_t stream) {
  PQ_TRY(check_score_call(e, a, images, scores));
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  return score_impl(e, a, images, false, scores, token_logprobs, reinterpret_cast<cudaStream_t>(stream));
}

int parseq_score_u8(parseq_engine* e, const parseq_score_args* a, const uint8_t* images_hwc, float* scores, float* token_logprobs,
                    parseq_stream_t stream) {
  PQ_TRY(check_score_call(e, a, images_hwc, scores));
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  return score_impl(e, a, images_hwc, true, scores, token_logprobs, reinterpret_cast<cudaStream_t>(stream));
}

int parseq_beam_search(parseq_engine* e, const parseq_beam_args* a, const float* images, int32_t* ids, int32_t* lengths,
                       float* scores, parseq_stream_t stream) {
  PQ_TRY(check_beam_call(e, a, images, ids, lengths, scores));
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  return beam_impl(e, a, images, false, ids, lengths, scores, reinterpret_cast<cudaStream_t>(stream));
}

int parseq_beam_search_u8(parseq_engine* e, const parseq_beam_args* a, const uint8_t* images_hwc, int32_t* ids,
                          int32_t* lengths, float* scores, parseq_stream_t stream) {
  PQ_TRY(check_beam_call(e, a, images_hwc, ids, lengths, scores));
  if (a->batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  return beam_impl(e, a, images_hwc, true, ids, lengths, scores, reinterpret_cast<cudaStream_t>(stream));
}

int parseq_lexicon_check(const parseq_config* cfg, const parseq_lexicon_desc* d) {
  if (cfg == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  return check_lexicon(d, cfg->num_tokens - 2, cfg->max_label_length);
}

int parseq_lexicon_create(parseq_engine* e, const parseq_lexicon_desc* d, parseq_lexicon** out, parseq_stream_t stream) {
  if (e == nullptr || out == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  PQ_TRY(check_lexicon(d, e->C, e->cfg.max_label_length));
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  auto* lx = new parseq_lexicon();
  lx->device = e->cfg.device; lx->C = e->C; lx->V = d->num_nodes; lx->E = d->num_edges;
  const long long E1 = std::max(d->num_edges, 1);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = lx->first_edge.alloc(lx->V + 1ll);
  if (rc == PARSEQ_OK) rc = lx->edge_class.alloc(E1);
  if (rc == PARSEQ_OK) rc = lx->edge_child.alloc(E1);
  if (rc == PARSEQ_OK) rc = lx->terminal.alloc(lx->V);
  auto up = [&](void* dst, const void* src, long long bytes) {
    if (rc == PARSEQ_OK && bytes > 0 && cudaMemcpyAsync(dst, src, static_cast<size_t>(bytes), cudaMemcpyHostToDevice, st) != cudaSuccess)
      rc = fail(PARSEQ_ERR_CUDA, "lexicon upload failed");
  };
  up(lx->first_edge, d->first_edge, 4ll * (lx->V + 1));
  up(lx->edge_class, d->edge_class, 4ll * lx->E);
  up(lx->edge_child, d->edge_child, 4ll * lx->E);
  up(lx->terminal, d->terminal, lx->V);
  if (rc == PARSEQ_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = fail(PARSEQ_ERR_CUDA, "lexicon upload failed");
  if (rc != PARSEQ_OK) {
    delete lx;
    return rc;
  }
  *out = lx;
  return PARSEQ_OK;
}

void parseq_lexicon_destroy(parseq_lexicon* lx) {
  if (lx == nullptr) return;
  cudaSetDevice(lx->device);
  delete lx;
}

int parseq_beam_search_lexicon(parseq_engine* e, const parseq_beam_args* a, const parseq_lexicon* lx, const int32_t* roots,
                               const float* images, int32_t* ids, int32_t* lengths, float* scores, parseq_stream_t stream) {
  return beam_lexicon_call(e, a, lx, roots, images, false, ids, lengths, scores, stream);
}

int parseq_beam_search_lexicon_u8(parseq_engine* e, const parseq_beam_args* a, const parseq_lexicon* lx,
                                  const int32_t* roots, const uint8_t* images_hwc, int32_t* ids, int32_t* lengths,
                                  float* scores, parseq_stream_t stream) {
  return beam_lexicon_call(e, a, lx, roots, images_hwc, true, ids, lengths, scores, stream);
}

int parseq_postprocess(const float* logits, int32_t batch, int32_t num_steps, int32_t num_classes, int32_t eos_id, int32_t* ids,
                       int32_t* lengths, float* confidence, parseq_stream_t stream) {
  if (logits == nullptr || ids == nullptr || lengths == nullptr || confidence == nullptr)
    return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (batch <= 0) return batch == 0 ? PARSEQ_OK : fail(PARSEQ_ERR_INVALID_ARG, "negative batch");
  pq::postprocess_kernel<<<(batch + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(logits, batch, num_steps, num_classes,
                                                                                              eos_id, ids, lengths, confidence);
  PQ_CUDA(cudaGetLastError());
  return PARSEQ_OK;
}

int parseq_encode(parseq_engine* e, int32_t batch, const float* images, float* memory, parseq_stream_t stream) {
  if (images == nullptr || memory == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  PQ_TRY(enter_main(e, user));
  const long long img_sz = 3ll * e->cfg.img_h * e->cfg.img_w;
  for (int b0 = 0; b0 < batch; b0 += e->chunk) {
    const int B = (batch - b0 < e->chunk) ? (batch - b0) : e->chunk;
    PQ_TRY(encode_chunk(e, images + b0 * img_sz, false, B, e->mem, memory + 1ll * b0 * e->T * e->D, e->main));
  }
  return leave_main(e, user);
}

int parseq_decode(parseq_engine* e, int32_t batch, int32_t ctx_len, int32_t num_queries, const int32_t* tgt, const float* memory,
                  const float* query, const uint8_t* query_mask, const uint8_t* padding_mask, float* out,
                  parseq_stream_t stream) {
  return parseq_decode_ex(e, batch, ctx_len, num_queries, tgt, memory, query, query_mask, padding_mask, nullptr, out, stream);
}

int parseq_decode_ex(parseq_engine* e, int32_t batch, int32_t ctx_len, int32_t num_queries, const int32_t* tgt,
                     const float* memory, const float* query, const uint8_t* query_mask, const uint8_t* padding_mask,
                     const uint8_t* content_mask, float* out, parseq_stream_t stream) {
  if (tgt == nullptr || memory == nullptr || out == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  if (e->arch != 0) return fail(PARSEQ_ERR_UNSUPPORTED, "decode: PARSeq only");
  if (batch < 0 || ctx_len < 1 || ctx_len > e->L || num_queries < 1 || num_queries > e->L)
    return fail(PARSEQ_ERR_INVALID_ARG, "decode: 1 <= context length, queries <= max_label_length + 1");
  if (batch == 0) return PARSEQ_OK;
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  PQ_TRY(enter_main(e, user));
  const int D = e->D, T = e->T, J = ctx_len, NQ = num_queries;
  parseq_engine::Stage& sg = e->stages[0];
  cudaStream_t st = e->main;
  for (int b0 = 0; b0 < batch; b0 += e->dec_chunk) {
    const int Bc = (batch - b0 < e->dec_chunk) ? (batch - b0) : e->dec_chunk;
    // memory (fp32, caller's) -> bf16 operand -> cross K/V cache rows [0, Bc * T)
    const long long n4 = 1ll * Bc * T * D / 4;
    pq::f32_to_bf16_kernel<<<static_cast<unsigned>(std::min<long long>((n4 + 255) / 256, 132ll * 8)), 256, 0, st>>>(
        reinterpret_cast<const float4*>(memory + 1ll * b0 * T * D), reinterpret_cast<uint2*>(e->mem.get()), n4);
    PQ_CUDA(cudaGetLastError());
    PQ_TRY(cross_kv(e, Bc));
    pq::copy_ids_kernel<<<(Bc * e->ids_ld + 255) / 256, 256, 0, st>>>(tgt + 1ll * b0 * J, J, sg.ids_ctx, Bc, e->ids_ld);
    PQ_CUDA(cudaGetLastError());
    e->launches += 2;
    DecodePass p;
    p.B = Bc; p.nq = NQ; p.nkeys = J; p.ids = sg.ids_ctx;
    p.query = query ? query + 1ll * b0 * NQ * D : nullptr;
    p.qmask = query_mask; p.cmask = content_mask;
    p.pmask = padding_mask ? padding_mask + 1ll * b0 * J : nullptr;
    p.tail = Tail::Norm; p.out_norm = out + 1ll * b0 * NQ * D;
    PQ_TRY(decode_pass(e, sg, p, st));
  }
  return leave_main(e, user);
}

int parseq_head(parseq_engine* e, int32_t rows, const float* x, float* logits, parseq_stream_t stream) {
  if (x == nullptr || logits == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_TRY(check_ready(e));
  if (rows <= 0) return rows == 0 ? PARSEQ_OK : fail(PARSEQ_ERR_INVALID_ARG, "negative rows");
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  cudaStream_t user = reinterpret_cast<cudaStream_t>(stream);
  PQ_TRY(enter_main(e, user));
  const int D = e->D;
  const int cap = e->dec_chunk * e->L;                 // rows of the bf16 staging buffer of a decoder chain
  parseq_engine::Stage& sg = e->stages[0];
  for (int r0 = 0; r0 < rows; r0 += cap) {
    const int n = (rows - r0 < cap) ? (rows - r0) : cap;
    const long long n4 = 1ll * n * D / 4;
    pq::f32_to_bf16_kernel<<<static_cast<unsigned>(std::min<long long>((n4 + 255) / 256, 132ll * 8)), 256, 0, e->main>>>(
        reinterpret_cast<const float4*>(x + 1ll * r0 * D), reinterpret_cast<uint2*>(sg.yn.get()), n4);
    PQ_CUDA(cudaGetLastError());
    e->launches++;
    e->cur_cat = CAT_DEC_GEMM;
    PQ_TRY(gemm(e, sg.yn, D, e->w("head.weight"), D, e->wf("head.bias"), n, e->C, D, pq::EPI_F32, 1.0f, nullptr, 0, 0,
                logits + 1ll * r0 * e->C, e->C, e->main));
  }
  return leave_main(e, user);
}

int parseq_text_embed(parseq_engine* e, int32_t n, const int32_t* ids, float* out, parseq_stream_t stream) {
  if (e == nullptr || ids == nullptr || out == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  if (e->arch != 0) return fail(PARSEQ_ERR_UNSUPPORTED, "text_embed: PARSeq only");
  if (n <= 0) return n == 0 ? PARSEQ_OK : fail(PARSEQ_ERR_INVALID_ARG, "negative count");
  if (!e->slots[e->index.at("text_embed.embedding.weight")].set) return fail(PARSEQ_ERR_STATE, "weights not set");
  PQ_CUDA(cudaSetDevice(e->cfg.device));
  const long long total = 1ll * n * e->D;
  pq::text_embed_kernel<<<static_cast<unsigned>(std::min<long long>((total + 255) / 256, 132ll * 8)), 256, 0,
                          reinterpret_cast<cudaStream_t>(stream)>>>(ids, e->wf("text_embed.embedding.weight"), out, n, e->D, e->V,
                                                                    std::sqrt(static_cast<float>(e->D)));
  PQ_CUDA(cudaGetLastError());
  return PARSEQ_OK;
}

int parseq_bench_tma_stream(void* buf, int64_t bytes, int cluster, int ctas, int nboxes, int nslot, int mode, void* sink,
                            parseq_stream_t stream) {
  if (buf == nullptr || sink == nullptr || cluster < 1 || cluster > 8 || ctas % cluster != 0 || nslot < 1 || nslot > 12)
    return fail(PARSEQ_ERR_INVALID_ARG, "bench_tma_stream: bad arguments");
  const long long rows_total = 8192;                         // rows per 64-column block
  const int blocks = static_cast<int>(bytes / (rows_total * 128));
  if (blocks < 1) return fail(PARSEQ_ERR_INVALID_ARG, "bench_tma_stream: buffer too small");
  PQ_TRY(ensure_kernel_attributes());
  CUtensorMap map;
  PQ_TRY(make_tmap3d(&map, buf, 64, rows_total, blocks, 64, 64 * rows_total, 64, 128));
  return launch_ex(LaunchConfig(dim3(static_cast<unsigned>(ctas)), dim3(pq::A2_THREADS + 32), kTmaBenchSmem,
                                reinterpret_cast<cudaStream_t>(stream), cluster > 1 ? static_cast<unsigned>(cluster) : 0, false),
                   pq::tma_stream_bench_kernel, map, nboxes, nslot, static_cast<int>(rows_total / 128), blocks, mode,
                   static_cast<unsigned int*>(sink));
}

int64_t parseq_debug_int(parseq_engine* e, const char* name) {
  if (name == nullptr) return -1;
  const std::string n(name);
  // launch options: per handle, or (NULL handle) those of the bare kernel exports; 0 until the first MODE 2 launch
  if (n == "ln_clusters") return (e ? e->lo : g_default_opts).ln_clusters;
  if (n == "live_device_bytes") return g_live_bytes;      // process-wide: every handle and lexicon
  if (n == "live_cuda_objects") return g_live_objects;
  if (e == nullptr) return -1;
  if (n == "ar2_occupancy_mt1_cs8") return e->ar2_occ[1][0];
  if (n == "ar2_occupancy_mt2_cs8") return e->ar2_occ[2][0];
  if (n == "ar2_occupancy_mt1_cs6") return e->ar2_occ[1][1];
  if (n == "ar2_occupancy_mt2_cs6") return e->ar2_occ[2][1];
  if (n == "ar_last_cluster_size") return e->ar_last_cs;
  if (n == "ar_last_per") return e->ar_last_per;
  if (n == "ar_last_clusters") return e->ar_last_ncl;
  if (n == "ar_last_mt") return e->ar_last_mt;
  if (n == "ar_last_head_split") return e->ar_last_hs;
  if (n == "ar_last_wide") return e->ar_last_wide;
  if (n == "ar_last_ids_pitch") return e->ar_last_idp;
  if (n == "ar_last_path") return e->ar_last_path;
  if (n == "sm_count") return e->lo.sm_count;
  if (n == "beam_bytes") return e->beam_bytes;
  if (n == "orient_rereads") return e->orient_rereads;
  if (n == "orient_readings") return e->orient_readings;
  return -1;
}
int64_t parseq_kernel_launches(const parseq_engine* e) { return e ? e->launches : 0; }

int parseq_set_option(parseq_engine* e, const char* name, int64_t value) {
  if (name == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null option");
  const std::string n(name);
  // launch options: per handle; with a NULL handle they set the process defaults used by the bare kernel exports
  // (parseq_gemm_bf16 & co.) and inherited by handles created afterwards
  LaunchOpts& lo = e ? e->lo : g_default_opts;
  // "block_n" and "cta_group" are accepted for compatibility and ignored: the GEMM has one 128 x 128 single-CTA tile
  if (n == "block_n") {
    if (value != 0 && value != 64 && value != 128 && value != 192 && value != 256)
      return fail(PARSEQ_ERR_INVALID_ARG, "block_n: 0/64/128/192/256");
    return PARSEQ_OK;
  }
  if (n == "cta_group") {
    if (value < 0 || value > 2) return fail(PARSEQ_ERR_INVALID_ARG, "cta_group: 0 (auto) / 1 / 2");
    return PARSEQ_OK;
  }
  if (n == "attn_impl") { lo.attn_impl = value != 0 ? 1 : 0; if (e) e->graphs.clear(); return PARSEQ_OK; }
  if (n == "pdl") { lo.use_pdl = value != 0; if (e) e->graphs.clear(); return PARSEQ_OK; }
  if (n == "gemm_stages") {
    // the MMA warpgroups release a stage once the next k-block's MMAs are queued: a ring needs at least two slots
    if (value < 0 || value == 1) return fail(PARSEQ_ERR_INVALID_ARG, "gemm_stages: 0 (full ring) or >= 2");
    lo.gemm_stages = static_cast<int>(value);
    if (e) e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "ln_cta_group") {
    if (value < 0 || value > 2) return fail(PARSEQ_ERR_INVALID_ARG, "ln_cta_group: 0 (auto) / 1 / 2");
    lo.ln_cta_group = static_cast<int>(value);
    if (e) e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "ln_split") {
    if (value < 0 || value > 2) return fail(PARSEQ_ERR_INVALID_ARG, "ln_split: 0 (auto) / 1 (off) / 2 (on)");
    lo.ln_split = static_cast<int>(value);
    if (e) e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "mlp_cta_group") {
    if (value < 0 || value > 2) return fail(PARSEQ_ERR_INVALID_ARG, "mlp_cta_group: 0 (auto) / 1 / 2");
    lo.mlp_cta_group = static_cast<int>(value);
    if (e) e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "pair_pdl") { lo.pair_pdl = value != 0; if (e) e->graphs.clear(); return PARSEQ_OK; }
  if (n == "fuse_mlp") {
    if (e == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null engine");
    e->fuse_mlp = value != 0 ? 1 : 0;
    e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "fuse_ln") {
    if (e == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null engine");
    e->fuse_ln = static_cast<int>(value) & 7;
    e->graphs.clear();
    return PARSEQ_OK;
  }
  if (e == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null engine");
  if (n == "timing") {
    e->timing = value != 0;
    for (auto& t : e->timed) { e->event_pool.push_back(std::move(t.a)); e->event_pool.push_back(std::move(t.b)); }
    e->timed.clear();
    return PARSEQ_OK;
  }
  if (n == "use_graph") { e->use_graph = value != 0; return PARSEQ_OK; }
  if (n == "ar_prof") { e->ar_prof_on = value != 0; e->graphs.clear(); return PARSEQ_OK; }
  if (n == "ar_clusters") {
    if (value < 0 || value > 1024) return fail(PARSEQ_ERR_INVALID_ARG, "ar_clusters out of range");
    e->ar_clusters_override = static_cast<int>(value);
    for (auto& r : e->ar2_clusters) r[0] = r[1] = 0;
    e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "ar_cluster_size") {
    if (value != 0 && value != 6 && value != 8) return fail(PARSEQ_ERR_INVALID_ARG, "ar_cluster_size: 0 (auto) / 6 / 8");
    e->ar_cs = static_cast<int>(value);
    e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "ar_kernel") {           // 0: AR loop as separate kernels, 1: grid-barrier kernel, 2: cluster kernel (ar_path)
    if (value < 0 || value > 2) return fail(PARSEQ_ERR_INVALID_ARG, "ar_kernel: 0 / 1 / 2");
    if (value == 1)
      if (const char* why = grid_barrier_limit(e)) return fail(PARSEQ_ERR_UNSUPPORTED, why);
    e->ar_kernel = static_cast<int>(value);
    e->graphs.clear();
    return PARSEQ_OK;
  }
  if (n == "chunk" || n == "max_batch" || n == "dec_chunk") {
    if (value <= 0 || value > 8192) return fail(PARSEQ_ERR_INVALID_ARG, "chunk / max_batch / dec_chunk out of range");
    // validate the new sizes BEFORE touching the workspace
    int chunk = e->chunk, dec_chunk = e->dec_chunk, max_batch = e->max_batch;
    if (n == "chunk") chunk = static_cast<int>(value);
    else if (n == "dec_chunk") dec_chunk = static_cast<int>(value);
    else { max_batch = static_cast<int>(value); chunk = max_batch; }
    if (chunk > max_batch) chunk = max_batch;
    if (dec_chunk > max_batch) dec_chunk = max_batch;
    if ((max_batch + dec_chunk - 1) / dec_chunk > 64) return fail(PARSEQ_ERR_INVALID_ARG, "too many decoder chains");
    PQ_CUDA(cudaSetDevice(e->cfg.device));
    PQ_CUDA(cudaDeviceSynchronize());
    const int old_chunk = e->chunk, old_dec = e->dec_chunk, old_max = e->max_batch;
    free_workspace(e);
    e->chunk = chunk; e->dec_chunk = dec_chunk; e->max_batch = max_batch;
    int r = alloc_workspace(e);
    if (r != PARSEQ_OK) {            // out of memory: back to the sizes that worked
      const std::string why = g_last_error;
      free_workspace(e);
      e->chunk = old_chunk; e->dec_chunk = old_dec; e->max_batch = old_max;
      if (alloc_workspace(e) != PARSEQ_OK) { e->finalized = false; free_workspace(e); e->broken = true; }
      return fail(r, why);
    }
    return PARSEQ_OK;
  }
  return fail(PARSEQ_ERR_INVALID_ARG, "unknown option: " + n);
}

int parseq_get_ar_profile(parseq_engine* e, uint64_t* out512) {
  if (e == nullptr || out512 == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "null argument");
  PQ_CUDA(cudaMemcpy(out512, e->ar_prof, 32 * 16 * 8, cudaMemcpyDeviceToHost));
  return PARSEQ_OK;
}

int parseq_get_timing(parseq_engine* e, int category, double* ms, double* flops, int64_t* count) {
  if (e == nullptr || category < 0 || category >= CAT_COUNT) return fail(PARSEQ_ERR_INVALID_ARG, "bad timing query");
  double tms = 0.0, tf = 0.0;
  int64_t n = 0;
  for (auto& t : e->timed) {
    if (t.cat != category) continue;
    float dt = 0.f;
    cudaError_t ce = cudaEventElapsedTime(&dt, t.a, t.b);
    if (ce != cudaSuccess) return fail(PARSEQ_ERR_CUDA, std::string("timing readback: ") + cudaGetErrorString(ce));
    tms += dt; tf += t.flops; ++n;
  }
  if (ms) *ms = tms;
  if (flops) *flops = tf;
  if (count) *count = n;
  return PARSEQ_OK;
}

int parseq_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias, int M, int N, int K,
                     int mode, float alpha, const float* resid, int64_t ldr, int resid_mod, void* out, int64_t ldo,
                     parseq_stream_t stream) {
  if (mode < 0 || mode > 2) return fail(PARSEQ_ERR_INVALID_ARG, "bad epilogue mode");
  PQ_TRY(ensure_kernel_attributes());
  return gemm_launch(g_default_opts, A, lda, W, ldw, bias, M, N, K, mode, alpha, resid, ldr, resid_mod, out, ldo,
                     reinterpret_cast<cudaStream_t>(stream));
}
int parseq_gemm_ln_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias, int M, int D, int K,
                         float* x_inout, const float* gamma, const float* beta, float eps, void* xn_bf16,
                         parseq_stream_t stream) {
  PQ_TRY(ensure_kernel_attributes());
  return gemm_ln_launch(g_default_opts, A, lda, W, ldw, bias, M, D, K, x_inout, gamma, beta, eps, xn_bf16, reinterpret_cast<cudaStream_t>(stream));
}
int parseq_mlp_ln_bf16(const void* xn, const void* W1, const float* b1, const void* W2, const float* b2, int M, int D,
                       float* x_inout, const float* gamma, const float* beta, float eps, void* xn_out_bf16, parseq_stream_t stream) {
  PQ_TRY(ensure_kernel_attributes());
  return mlp_ln_launch(g_default_opts, xn, W1, b1, W2, b2, M, D, x_inout, gamma, beta, eps, xn_out_bf16,
                       reinterpret_cast<cudaStream_t>(stream));
}
int parseq_layernorm_bf16(const float* x, const float* gamma, const float* beta, float eps, int M, int D, void* y_bf16,
                          float* y_f32_or_null, parseq_stream_t stream) {
  PQ_TRY(ensure_kernel_attributes());
  return layernorm_launch(g_default_opts, x, gamma, beta, eps, M, D, y_bf16, y_f32_or_null, reinterpret_cast<cudaStream_t>(stream));
}
int parseq_enc_attention(const void* qkv_bf16, int B, int T, int D, int heads, void* out_bf16, parseq_stream_t stream) {
  PQ_TRY(ensure_kernel_attributes());
  PQ_TRY(ensure_sm_count(g_default_opts));
  return enc_attention_launch(g_default_opts, qkv_bf16, B, T, D, heads, out_bf16, reinterpret_cast<cudaStream_t>(stream));
}
int parseq_qkv_attention_bf16(const void* xn_bf16, const void* W_qkv, const float* b_qkv, int B, int T, int D, int heads,
                              void* out_bf16, parseq_stream_t stream) {
  PQ_TRY(ensure_kernel_attributes());
  return qkv_attn_launch(g_default_opts, xn_bf16, W_qkv, b_qkv, B, T, D, heads, out_bf16, reinterpret_cast<cudaStream_t>(stream));
}
int parseq_head_lse_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias, int M, int N, int K,
                         const int32_t* tgt, float* part, float* tlogit, parseq_stream_t stream) {
  if (part == nullptr || (tgt == nullptr) != (tlogit == nullptr))
    return fail(PARSEQ_ERR_INVALID_ARG, "head_lse: part is required, tgt and tlogit go together");
  PQ_TRY(ensure_kernel_attributes());
  return gemm_lse_launch(g_default_opts, A, lda, W, ldw, bias, M, N, K, tgt, reinterpret_cast<float2*>(part), tlogit,
                         reinterpret_cast<cudaStream_t>(stream));
}
int parseq_head_topk_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias, int M, int N, int K,
                          int k, const uint32_t* mask, int mask_div, float* part, uint64_t* keys, parseq_stream_t stream) {
  if (k < 1 || k > pq::BEAM_TOPK_LD) return fail(PARSEQ_ERR_INVALID_ARG, "head_topk: k must be in 1..16");
  if (part == nullptr || keys == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "head_topk: part and keys are required");
  if (mask != nullptr && mask_div < 1) return fail(PARSEQ_ERR_INVALID_ARG, "head_topk: mask_div must be >= 1");
  PQ_TRY(ensure_kernel_attributes());
  return gemm_topk_launch(g_default_opts, A, lda, W, ldw, bias, M, N, K, k, mask, mask != nullptr ? mask_div : 1,
                          reinterpret_cast<float2*>(part), reinterpret_cast<unsigned long long*>(keys),
                          reinterpret_cast<cudaStream_t>(stream));
}
int parseq_beam_select(const parseq_beam_select_args* a, parseq_stream_t stream) {
  if (a == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: null arguments");
  const int C = a->num_classes, K = a->beam_width;
  const bool lex = a->first_edge != nullptr;
  if (a->batch < 1 || C < 1) return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: batch and num_classes must be >= 1");
  if (K < 1 || K > pq::BEAM_MAX) return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: beam_width must be in 1..16");
  if (a->ntiles != (C + pq::GEMM_BLOCK_N - 1) / pq::GEMM_BLOCK_N)
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: ntiles must be ceil(num_classes / 128)");
  if (a->step < 0 || a->step >= a->num_steps) return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: need 0 <= step < num_steps");
  if (a->ids_ld <= a->num_steps) return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: ids_ld must exceed num_steps");
  if (a->logits == nullptr && (a->keys == nullptr || lex))
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: logits are required without keys and with a lexicon");
  if (a->keys != nullptr && a->part == nullptr) return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: keys need part");
  if (a->class_mask != nullptr && a->mask_ld < (C + 31) / 32)
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: mask_ld must be >= ceil(num_classes / 32)");
  if (a->ids_in == nullptr || a->score_in == nullptr || a->len_in == nullptr || a->st_in == nullptr || a->ids_out == nullptr ||
      a->score_out == nullptr || a->len_out == nullptr || a->st_out == nullptr || a->parent == nullptr ||
      (a->step + 1 == a->num_steps && (a->out_ids == nullptr || a->out_len == nullptr || a->out_score == nullptr)))
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: missing state or output array");
  if (lex && (a->edge_class == nullptr || a->edge_child == nullptr || a->terminal == nullptr || a->node_out == nullptr ||
              (a->step > 0 && a->node_in == nullptr)))
    return fail(PARSEQ_ERR_INVALID_ARG, "beam_select: incomplete lexicon");
  PQ_TRY(ensure_kernel_attributes());
  pq::BeamLex bl{};
  if (lex) bl = pq::BeamLex{a->first_edge, a->edge_class, a->edge_child, a->terminal, a->roots, a->node_in, a->node_out};
  return launch_k(g_default_opts, lex ? pq::beam_select_kernel<true> : pq::beam_select_kernel<false>,
                  dim3(static_cast<unsigned>(a->batch)), dim3(pq::BEAM_THREADS), 0, reinterpret_cast<cudaStream_t>(stream),
                  a->logits, reinterpret_cast<const float2*>(a->part),
                  reinterpret_cast<const unsigned long long*>(lex ? nullptr : a->keys), a->ntiles, static_cast<long long>(a->row0),
                  static_cast<long long>(a->img_stride), static_cast<long long>(a->slot_stride), C, K, a->step, a->num_steps,
                  a->class_mask, a->mask_ld, a->ids_in, a->score_in, a->len_in, a->st_in, a->ids_out, a->score_out, a->len_out,
                  a->st_out, a->parent, a->ids_ld, a->out_ids, a->out_len, a->out_score, bl);
}

}  // extern "C"

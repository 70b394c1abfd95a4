// Cluster-owned autoregressive decode: the whole `decode_ar` loop of PARSeq.forward (model.py:119-147) with NO
// device-wide synchronisation.  One thread-block cluster (8 CTAs) owns up to 32 images for all L steps; clusters never
// talk to each other, so the kernel needs no co-residency guarantee (the v1 kernel, dec_ar.cuh, used 8 software grid
// barriers per step over 148 CTAs), may share the GPU with any other work, and its critical path per step is a chain
// of hardware cluster barriers (~0.2 us) instead of grid barriers (~1.7 us) plus re-partitioned phases.
//
// Work split inside a cluster (rank k of 8, rows = images of the cluster, D = embed dim, DS = D/8):
//   * every projection is split over N: CTA k computes output columns [k*DS, (k+1)*DS) for ALL rows on mma.sync
//     tiles; the weight slice streams through a ring of 16 KB shared-memory slots filled by TMA (128B-swizzled boxes,
//     one elected thread issues the next box whenever a slot is released): each weight byte is read from L2 once per
//     cluster and step;
//   * attention is split over images: CTA k owns rows k, k+8, ... ; cross-attention streams the image's K/V cache
//     (T x 2D bf16) through the same ring and runs QK^T / PV as block-diagonal tensor-core products
//     (rows = heads; q and P are split into bf16 hi + lo terms, i.e. ~16 mantissa bits);
//   * the fp32 residual stream y lives column-sliced in the owning CTA; LayerNorm exchanges per-slice (mean, M2)
//     through distributed shared memory (Chan merge in fixed order, identical in every CTA) and all-gathers the
//     normalised bf16 rows, which are the A operand of the next projection;
//   * linear2 is split over K (each CTA multiplies the hidden slice it just produced), partial sums are
//     scattered to the column owners and added in fixed order (deterministic, batch-invariant);
//   * the character head runs redundantly in every CTA, so every CTA derives the same greedy token locally - up to 96
//     classes.  Larger heads (WIDE, > 128 classes) are split over the cluster: CTA k owns the classes
//     [k*Cs, (k+1)*Cs), streams only that slice of head.weight through the ring in [128 x 64] boxes, stores its logits
//     straight from the MMA fragments and exchanges one (max, lowest index) pair per row through distributed shared
//     memory; every CTA merges the pairs in rank order (= class order), so all derive the same token, the first maximum
//     as torch.argmax picks it.
// Numerics: bf16 tensor-core operands, fp32 accumulation, fp32 residual / LayerNorm / softmax statistics, exact-erf
// GELU polynomial (ptx.cuh) - the rounding points of the v1 kernel and of the multi-kernel path.
#pragma once
#include <cuda.h>

#include "ptx.cuh"

namespace pq {

struct DecAr2Maps {
  CUtensorMap wo_s, wq_c, wo_c, w1, w2, wh, ckv;
};

struct DecAr2Params {
  int B, L, V, C, T, per;         // per = images per cluster
  int tbox, tb;                   // K/V box rows (64 or 128) and number of 128-key blocks
  float qscale;
  const float* qs;                // [L, D] pre-scaled self-attention queries of pos_queries
  const __nv_bfloat16* kvtab;     // [(pos*V + tok), 2D]
  const float* posq;              // [L, D]
  const float *bo_s, *bq_c, *bo_c, *b1, *b2, *bh;
  const float *g1, *be1, *g2, *be2, *g3, *be3;
  int* ids;                       // [B, ids_ld]: ids[:,0] = BOS on entry; filled on exit
  int ids_ld;
  float* logits;                  // [B, L, C]
  const int* forced;              // optional teacher forcing [B, forced_ld]
  int forced_ld;
  const uint32_t* mask;           // optional class allowlist [B, ceil(C / 32)] words (ptx.cuh class_allowed)
  unsigned long long* prof;       // optional [32][16] globaltimer stamps of cluster 0 / rank 0, or nullptr (A2_PROF)
};

constexpr int A2_THREADS = 256;      // consumer threads (warps 0-7)
constexpr int A2_LAUNCH_THREADS = 288;   // + warp 8: the TMA producer
constexpr int A2_SLOT = 16384;      // ring slot bytes
constexpr int A2_SLOG_LD = 104;     // fp32 row pitch of the staged logits
constexpr int A2_PROF_STEPS = 26;   // steps with a row of their own in the [32][16] profile buffer (row 26: step 1 extras)

__device__ __forceinline__ void cluster_sync_relacq() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
// named barriers: 1 = the 8 consumer warps; 2 + s = "slot s is free" (consumers arrive, the producer warp waits)
__device__ __forceinline__ void a2_csync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void a2_slot_arrive(int s) { asm volatile("bar.arrive %0, 288;" ::"r"(2 + s) : "memory"); }
__device__ __forceinline__ void a2_slot_wait(int s) { asm volatile("bar.sync %0, 288;" ::"r"(2 + s) : "memory"); }
__device__ __forceinline__ void st_cluster_v4(uint32_t addr, uint4 v) {
  asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_cluster_v2f(uint32_t addr, float a, float b) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ unsigned long long a2_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// byte offset of (row r, bf16 column c) in an A-operand buffer made of [ROWS x 64] 128B-swizzled tiles
template <int ROWS>
__device__ __forceinline__ uint32_t a_off(int r, int c) {
  return static_cast<uint32_t>((c >> 6) * (ROWS * 128) + r * 128 + (((((c & 63) >> 3) ^ (r & 7)) << 4) | ((c & 7) << 1)));
}
// byte offset of (row r, bf16 column c < 64) inside one swizzled box
__device__ __forceinline__ uint32_t box_off(int r, int c) {
  return static_cast<uint32_t>(r * 128 + ((((c >> 3) ^ (r & 7)) << 4) | ((c & 7) << 1)));
}

// IDP: row pitch of the per-cluster id buffer s_ids, 32 (L <= 32) or 64 (L <= 64 decode positions)
template <int D, int MT, int CS_, int IDP = 32>
struct A2Cfg {
  static constexpr int CS = CS_;                       // CTAs per cluster (8; 6 can pack more SMs of a GPC)
  static constexpr int ROWS = 16 * MT;                 // rows (images) per cluster, padded
  static constexpr int OWN = (ROWS + CS - 1) / CS;     // rows owned by one CTA for the attention phases
  static constexpr int DS = D / CS;                    // column slice of a D-wide projection
  static constexpr int MD = 4 * D;                     // decoder MLP width (dec_mlp_ratio = 4)
  static constexpr int MS = MD / CS;                   // hidden slice
  static constexpr int KT = D / 64;                    // 64-wide k-blocks of a D-deep product
  static constexpr int KT2 = (MS + 63) / 64;           // k-blocks of the linear2 slice
  static constexpr int H = D / 32;                     // decoder heads (head_dim 32)
  static constexpr int MH = (H + 15) / 16;             // m16 tiles over the heads
  static constexpr int G = 8 / MT;                     // warp groups along N
  static constexpr int NC1 = (MS % 128 == 0) ? 128 : 96;   // linear1 N-chunk rows (MS = 96 / 192 / 384)
  static constexpr int NCH1 = MS / NC1;
  static constexpr int NC2 = (D % 128 == 0) ? 128 : 96;    // linear2 N-chunk rows (D = 192 / 384 / 768)
  static constexpr int NCH2 = D / NC2;
  static constexpr int GS = (A2_SLOT / (DS * 128) < KT) ? (A2_SLOT / (DS * 128)) : KT;   // k-blocks of a DS-row slice per slot
  static constexpr int NSL_S = (KT + GS - 1) / GS;     // slots per D x D slice
  // ---- shared memory map (bytes) ----
  static constexpr int A_BYTES = KT * ROWS * 128;      // one A buffer [ROWS, D] bf16
  static constexpr int R_BYTES = ROWS * D * 4;         // a2 (first half) aliased with the linear2 receive buffer
  static constexpr int HD_BYTES = KT2 * ROWS * 128;
  static constexpr int Y_BYTES = ROWS * DS * 4;
  static constexpr int Q_BYTES = OWN * D * 4;
  static constexpr int P_BYTES = 2 * MH * 16 * 256 * 2;   // P hi + lo, [16 MH, 256 keys] bf16
  static constexpr int CA_BYTES = D * 2;
  static constexpr int ST_BYTES = CS * ROWS * 8;
  static constexpr int RED_BYTES = 2 * 8 * MH * 16 * 4;
  static constexpr int IDS_BYTES = ROWS * IDP * 4;
  static constexpr int SLOG_BYTES = ROWS * A2_SLOG_LD * 4;
  static constexpr int MISC_BYTES = 1024;              // mbarriers, row statistics
  static constexpr int PART_BYTES = 8 * D * 4;         // cross-attention partial outputs of the 8 key slices (one image)
  static constexpr int QF_BYTES = KT * 16 * 16;        // bf16 hi / lo A-fragment words of one image's cross-attention query
  static constexpr int PL_BYTES = P_BYTES > SLOG_BYTES ? P_BYTES : SLOG_BYTES;   // P (cross-attention) and the staged logits (head) share
  static constexpr int FIXED = A_BYTES + R_BYTES + HD_BYTES + Y_BYTES + Q_BYTES + PL_BYTES + CA_BYTES + ST_BYTES + RED_BYTES +
                               IDS_BYTES + MISC_BYTES + QF_BYTES + PART_BYTES + ROWS * 8;
  static constexpr int NSLOT_RAW = (232448 - 1024 - FIXED) / A2_SLOT;
  static constexpr int NSLOT = NSLOT_RAW > 8 ? 8 : NSLOT_RAW;
  static constexpr int SMEM = 1024 + NSLOT * A2_SLOT + FIXED;
  static_assert(NSLOT >= 3, "ring too shallow");
  static_assert(IDP == 32 || IDP == 64, "id row pitch");
  static_assert(D % CS == 0 && DS % 8 == 0 && MS % 32 == 0, "slices");
  static_assert(DS * 128 <= A2_SLOT && NC1 * 128 <= A2_SLOT && NC2 * 128 <= A2_SLOT, "box fits a slot");
};

template <int D, int MT, int CS, int IDP = 32>
constexpr size_t dec_ar2_smem_bytes() { return static_cast<size_t>(A2Cfg<D, MT, CS, IDP>::SMEM); }

// ------------------------------------------------------------------------------------------------------------------
// TMA ring: a static per-step program of slot fills; one thread issues, everybody consumes in program order.
// WIDE: the head segment is this CTA's class slice, ceil(Cs / 128) chunks of KT [128 x 64] boxes.
template <int D, int MT, int CS, bool WIDE = false, int IDP = 32>
struct A2Ring {
  using Cfg = A2Cfg<D, MT, CS, IDP>;
  uint8_t* slots;
  uint64_t* full;
  const DecAr2Maps* maps;
  int rank, n_own, img0, per_here;     // img0: first image of the cluster
  int hs_row, hs_kb;                   // head-split mode (few images per cluster): this CTA's (row, k-block) unit, or hs_row < 0
  int tbox, tb, T;
  int items_per_step, total;
  int seg_b, seg_c, seg_d, seg_e, seg_f, seg_g;   // first item index of each segment
  int cons, prod;
  int head_row0, head_rows;            // WIDE: first class of this CTA's slice, number of classes C

  // n_kv_units: (image, k-block) cross-attention units of this CTA: n_own * KT, or 0 / 1 in head-split mode
  // head_chunks (WIDE): 128-class chunks of this CTA's slice
  __device__ void init(uint8_t* slots_, uint64_t* full_, const DecAr2Maps* maps_, int rank_, int n_own_, int img0_, int tbox_,
                       int tb_, int T_, int steps, int n_kv_units, int hs_row_, int hs_kb_, int head_chunks = 0,
                       int head_row0_ = 0, int head_rows_ = 0) {
    slots = slots_; full = full_; maps = maps_; rank = rank_; n_own = n_own_; img0 = img0_; tbox = tbox_; tb = tb_; T = T_;
    hs_row = hs_row_; hs_kb = hs_kb_;
    seg_b = Cfg::NSL_S;
    seg_c = 2 * Cfg::NSL_S;
    seg_d = seg_c + n_kv_units * 2 * tb;
    seg_e = seg_d + Cfg::NSL_S;
    seg_f = seg_e + Cfg::NCH1 * Cfg::KT;
    seg_g = seg_f + Cfg::NCH2 * Cfg::KT2;
    if constexpr (WIDE) {
      items_per_step = seg_g + head_chunks * Cfg::KT;
      head_row0 = head_row0_; head_rows = head_rows_;
    } else {
      items_per_step = seg_g + Cfg::KT;
    }
    total = items_per_step * steps;
    cons = 0; prod = 0;
  }
  // D x D slice item j: k-blocks [j*GS, ...) of rows [rank*DS, +DS)
  __device__ void issue_slice(const CUtensorMap* m, int j, uint8_t* dst, uint64_t* bar) {
    const int k0 = j * Cfg::GS;
    const int n = (Cfg::KT - k0 < Cfg::GS) ? (Cfg::KT - k0) : Cfg::GS;
    mbar_expect_tx(bar, static_cast<uint32_t>(n * Cfg::DS * 128));
    for (int i = 0; i < n; ++i) tma_load_2d(dst + i * Cfg::DS * 128, m, bar, (k0 + i) * 64, rank * Cfg::DS);
  }
  __device__ void issue(int it, int s) {       // one thread; it = item index inside the step, s = slot
    uint8_t* dst = slots + s * A2_SLOT;
    uint64_t* bar = &full[s];
    if (it < seg_b) { issue_slice(&maps->wo_s, it, dst, bar); return; }
    if (it < seg_c) { issue_slice(&maps->wq_c, it - seg_b, dst, bar); return; }
    if (it < seg_d) {                    // K/V boxes: (own image, K|V, k-block, key block)
      int j = it - seg_c;
      const int t = j % tb; j /= tb;
      int kb, kv, img;
      if (hs_row >= 0) {                 // head-split: one (image, k-block) unit: K boxes, then V boxes
        kb = hs_kb; kv = j & 1; img = img0 + hs_row;
      } else {
        kb = j % Cfg::KT; j /= Cfg::KT;
        kv = j & 1;
        img = img0 + rank + CS * (j >> 1);
      }
      // column-blocked cache [2D/64][max_batch][T][64] (engine.cu make_tmap_kv4d): keys t*128 .. of this image only;
      // keys past T are zero-filled, and the fill counts towards the box's tx bytes
      mbar_expect_tx(bar, static_cast<uint32_t>(tbox * 128));
      tma_load_4d(dst, &maps->ckv, bar, 0, t * 128, img, kv * Cfg::KT + kb);
      return;
    }
    if (it < seg_e) { issue_slice(&maps->wo_c, it - seg_d, dst, bar); return; }
    if (it < seg_f) {                    // linear1: chunk c (NC1 rows of this CTA's hidden slice), k-block kb
      const int j = it - seg_e, c = j / Cfg::KT, kb = j % Cfg::KT;
      mbar_expect_tx(bar, Cfg::NC1 * 128);
      tma_load_2d(dst, &maps->w1, bar, kb * 64, rank * Cfg::MS + c * Cfg::NC1);
      return;
    }
    if (it < seg_g) {                    // linear2: output chunk c (NC2 rows of W2), k-block kb of this CTA's K slice
      const int j = it - seg_f, c = j / Cfg::KT2, kb = j % Cfg::KT2;
      mbar_expect_tx(bar, Cfg::NC2 * 128);
      tma_load_2d(dst, &maps->w2, bar, rank * Cfg::MS + kb * 64, c * Cfg::NC2);
      return;
    }
    if constexpr (WIDE) {                // head chunk c: classes [head_row0 + 128 c, +128), k-block kb
      const int j = it - seg_g, c = j / Cfg::KT, kb = j % Cfg::KT;
      // rows >= C are zero-filled by the tensor map bounds; a chunk that starts past C (an empty tail slice) reads
      // in-bounds rows instead and none of its columns is used
      const int row = head_row0 + c * 128;
      mbar_expect_tx(bar, 128 * 128);
      tma_load_2d(dst, &maps->wh, bar, kb * 64, row < head_rows ? row : head_rows - 1);
    } else {
      mbar_expect_tx(bar, 96 * 128);     // head: [96 x 64] (row 95.. zero-filled by the tensor map bounds)
      tma_load_2d(dst, &maps->wh, bar, (it - seg_g) * 64, 0);
    }
  }
  // ---- producer warp (warp 8): issues every item in program order; item i >= NSLOT waits on the named barrier of its
  //      slot until the 256 consumer threads have arrived there after item i - NSLOT
  int prod_it, prod_slot;
  __device__ void producer_begin() { prod = 0; prod_it = 0; prod_slot = 0; }
  __device__ __forceinline__ void produce(int n) {            // all 32 lanes of the producer warp
    for (int k = 0; k < n; ++k) {
      if (prod >= Cfg::NSLOT) a2_slot_wait(prod_slot);
      if ((threadIdx.x & 31) == 0) issue(prod_it, prod_slot);
      __syncwarp();
      ++prod;
      if (++prod_it == items_per_step) prod_it = 0;
      if (++prod_slot == Cfg::NSLOT) prod_slot = 0;
    }
  }
  // ---- consumer warps: no CTA-wide barrier per item
  __device__ __forceinline__ const uint8_t* wait() {          // one lane per warp polls the barrier
    const int s = cons % Cfg::NSLOT;
    if ((threadIdx.x & 31) == 0) mbar_wait(&full[s], static_cast<uint32_t>((cons / Cfg::NSLOT) & 1));
    __syncwarp();
    return slots + s * A2_SLOT;
  }
  __device__ __forceinline__ void release() {                  // this warp is done reading the slot
    if (cons + Cfg::NSLOT < total) a2_slot_arrive(cons % Cfg::NSLOT);   // (the last NSLOT items are never refilled)
    ++cons;
  }
};

// acc[j] (+)= A[mi-th 16 rows, 64 k of tile `atile`] * Box[n rows, 64 k]^T for this warp's NTW n8-tiles starting at n8
// tile `nt0`; A tile and box are 128B-swizzled [rows][64].
template <int NTW>
__device__ __forceinline__ void mma_box(float (&acc)[NTW][4], const uint8_t* atile, int mi, const uint8_t* box, int nt0,
                                        int lane, int ksteps = 4) {
  // Every n8 tile accumulates its even and odd k-steps in separate registers (two independent dependency chains per
  // box: the phases are latency-, not throughput-bound); the odd chain is folded into `acc` before returning.
  const uint32_t abase = smem_u32(atile), bbase = smem_u32(box);
  float odd[NTW][4];
#pragma unroll
  for (int j = 0; j < NTW; ++j) odd[j][0] = odd[j][1] = odd[j][2] = odd[j][3] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    if (ks < ksteps) {
      uint32_t a0, a1, a2, a3;
      ldmatrix_x4(abase + box_off(mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, ks * 16 + (lane >> 4) * 8), a0, a1, a2, a3);
#pragma unroll
      for (int np = 0; np < NTW / 2; ++np) {
        const int n = (nt0 + np * 2) * 8 + (lane & 7) + (lane >> 4) * 8;
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(bbase + box_off(n, ks * 16 + ((lane >> 3) & 1) * 8), b0, b1, b2, b3);
        if (ks & 1) {
          mma_bf16_16816(odd[np * 2], a0, a1, a2, a3, b0, b1);
          mma_bf16_16816(odd[np * 2 + 1], a0, a1, a2, a3, b2, b3);
        } else {
          mma_bf16_16816(acc[np * 2], a0, a1, a2, a3, b0, b1);
          mma_bf16_16816(acc[np * 2 + 1], a0, a1, a2, a3, b2, b3);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < NTW; ++j) {
    acc[j][0] += odd[j][0]; acc[j][1] += odd[j][1]; acc[j][2] += odd[j][2]; acc[j][3] += odd[j][3];
  }
}

// HS: head-split cross-attention (launch-wide: rows per cluster x k-blocks <= cluster size; see below).  A template flag
// so that the throughput instantiations carry none of its registers / branches.
// WIDE: the class-sliced head for C > 128 (see the top of the file); `maps.wh` then has [128 x 64] boxes.  The body is
// shared by two kernels, dec_ar2_kernel (WIDE = false) and dec_ar2_wide_kernel (WIDE = true).
template <int D, int MT, int CS, bool HS, bool WIDE, int IDP>
__device__ __forceinline__ void dec_ar2_body(const DecAr2Maps& maps, const DecAr2Params p) {
  using Cfg = A2Cfg<D, MT, CS, IDP>;
  constexpr int ROWS = Cfg::ROWS, DS = Cfg::DS, KT = Cfg::KT, KT2 = Cfg::KT2, MS = Cfg::MS, MH = Cfg::MH, G = Cfg::G,
                OWN = Cfg::OWN, H = Cfg::H;
  extern __shared__ uint8_t a2_smem_raw[];
  const uint32_t raw = smem_u32(a2_smem_raw);
  uint8_t* sm = a2_smem_raw + (((raw + 1023u) & ~1023u) - raw);
  uint8_t* s_ring = sm;                                         sm += Cfg::NSLOT * A2_SLOT;
  uint8_t* s_a1 = sm;                                           sm += Cfg::A_BYTES;
  uint8_t* s_a2 = sm;          /* recv aliases a2 */            sm += Cfg::R_BYTES;
  float* s_recv = reinterpret_cast<float*>(s_a2);               // [8 src][ROWS][DS]
  uint8_t* s_hd = sm;                                           sm += Cfg::HD_BYTES;
  float* s_y = reinterpret_cast<float*>(sm);                    sm += Cfg::Y_BYTES;     // [ROWS][DS]
  float* s_q = reinterpret_cast<float*>(sm);                    sm += Cfg::Q_BYTES;     // [OWN][D]
  uint8_t* s_p = sm;                                            sm += Cfg::PL_BYTES;    // hi | lo; the head stages its logits here
  __nv_bfloat16* s_ca = reinterpret_cast<__nv_bfloat16*>(sm);   sm += Cfg::CA_BYTES;
  float2* s_st = reinterpret_cast<float2*>(sm);                 sm += Cfg::ST_BYTES;    // [8 src][ROWS] (mean, M2)
  float* s_red = reinterpret_cast<float*>(sm);                  sm += Cfg::RED_BYTES;   // [2][8 warps][16 MH]
  int* s_ids = reinterpret_cast<int*>(sm);                      sm += Cfg::IDS_BYTES;   // [ROWS][IDP]
  float* s_log = reinterpret_cast<float*>(s_p);
  float2* s_mr = reinterpret_cast<float2*>(sm);                 sm += ROWS * 8;         // per row (mean, rstd)
  uint4* s_qf = reinterpret_cast<uint4*>(sm);                   sm += Cfg::QF_BYTES;    // [KT][4 k-steps][4 t]: hi01, hi89, lo01, lo89
  float* s_part = reinterpret_cast<float*>(sm);                 sm += Cfg::PART_BYTES;  // [8 warps][D]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(sm);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int rank = static_cast<int>(cluster_ctarank());
  const int cl = blockIdx.x / CS;
  const int img0 = cl * p.per;
  const int nrows = (p.B - img0 < p.per) ? (p.B - img0) : p.per;    // images of this cluster (>= 1)
  const int n_own = (nrows > rank) ? ((nrows - rank + CS - 1) / CS) : 0;
  const int mi = warp / G, ng = warp % G;                            // GEMM warp tiling: m16 tile, n group

  grid_dep_launch();
  if (tid == 0) {
    for (int s = 0; s < Cfg::NSLOT; ++s) mbar_init(&s_bar[s], 1);
    fence_mbar_init();
    prefetch_tmap(&maps.wo_s); prefetch_tmap(&maps.wq_c); prefetch_tmap(&maps.wo_c); prefetch_tmap(&maps.w1);
    prefetch_tmap(&maps.w2); prefetch_tmap(&maps.wh); prefetch_tmap(&maps.ckv);
  }
  // zero the A buffers once: padded rows (>= nrows) are multiplied but never stored; keep them finite
  for (int i = tid; i < (Cfg::A_BYTES + Cfg::R_BYTES + Cfg::HD_BYTES) / 16; i += A2_LAUNCH_THREADS)
    reinterpret_cast<uint4*>(s_a1)[i] = make_uint4(0u, 0u, 0u, 0u);
  grid_dep_wait();                    // weights / K/V cache / ids of the producing kernels are visible from here on
  for (int i = tid; i < ROWS * IDP; i += A2_LAUNCH_THREADS) {
    const int r = i >> (IDP == 32 ? 5 : 6), c = i & (IDP - 1);
    s_ids[i] = (r < nrows) ? p.ids[static_cast<long long>(img0 + r) * p.ids_ld + c] : 0;
  }
  // Head-split cross-attention: with so few images that (images x 64-channel k-blocks) fit the cluster, every CTA takes ONE
  // (image, k-block = head pair) unit instead of whole images - at bs = 1 six CTAs stream one K and one V panel each instead of
  // one CTA streaming twelve.  Per head the arithmetic and its order are unchanged (same bits as the image-split path).
  constexpr bool hs = HS;                                            // (the host launches HS only if p.per * KT <= CS)
  const int hs_row = (hs && rank < nrows * KT) ? rank / KT : -1;
  const int hs_kb = hs ? rank % KT : 0;
  const int c_own = hs ? (hs_row >= 0 ? 1 : 0) : n_own;             // cross-attention passes of this CTA
  A2Ring<D, MT, CS, WIDE, IDP> ring;
  // WIDE: classes per CTA, a multiple of 8 (whole n8 tiles); the last slices may be short or empty
  const int h_cs = WIDE ? (((p.C + CS - 1) / CS + 7) & ~7) : 0;
  const int h_chunks = (h_cs + 127) / 128;
  ring.init(s_ring, s_bar, &maps, rank, n_own, img0, p.tbox, p.tb, p.T, p.L, hs ? c_own : n_own * KT, hs ? hs_row : -1, hs_kb,
            h_chunks, rank * h_cs, p.C);
  __syncthreads();
  cluster_sync_relacq();              // every CTA of the cluster is running (remote stores are legal) and zero-filled

  if (warp == 8) {
    // ===================== TMA producer warp =====================
    // Issues the step's items in program order, each as soon as its slot is free.  It joins every cluster barrier of
    // the consumers, but arrives early and waits late (it touches no exchanged data), so that it runs up to one barrier
    // interval ahead of them: the items of a phase are in flight while the consumers are still in the previous one.
    ring.producer_begin();
    bool pending = false;
    auto csync_p = [&]() {
      if (pending) cluster_wait_acquire();
      cluster_arrive_release();
      pending = true;
    };
    const int n_kv = ring.seg_d - ring.seg_c;
    for (int step = 0; step < p.L; ++step) {
      csync_p();                                                   // (1)
      ring.produce(Cfg::NSL_S);                                    // P2: self-attention out-projection slice
      csync_p();                                                   // (2)
      csync_p();                                                   // (3)
      ring.produce(Cfg::NSL_S);                                    // P3: cross-attention query-projection slice
      csync_p();                                                   // (4)
      ring.produce(n_kv);                                          // P4: K / V panels of the owned images
      csync_p();                                                   // (5)
      ring.produce(Cfg::NSL_S);                                    // P5: cross-attention out-projection slice
      csync_p();                                                   // (6)
      csync_p();                                                   // (7)
      ring.produce(Cfg::NCH1 * KT + Cfg::NCH2 * KT2);              // P6 + P7: linear1 / linear2 slices
      csync_p();                                                   // (8)
      csync_p();                                                   // (9)
      csync_p();                                                   // (10)
      if constexpr (WIDE) {
        ring.produce(h_chunks * KT);                               // P8: this CTA's head slice
        csync_p();                                                 // (11) argmax pairs exchanged
      } else {
        ring.produce(KT);                                          // P8: head
      }
    }
    if (pending) cluster_wait_acquire();
  } else {

  // ---- helpers -------------------------------------------------------------------------------------------------
  // all-gather 8 bf16 columns (16 B) of row r into `buf` of every CTA of the cluster
  auto bcast16 = [&](uint8_t* buf, int r, int c, uint4 v) {
    const uint32_t off = smem_u32(buf) + a_off<ROWS>(r, c);
#pragma unroll
    for (int pe = 0; pe < CS; ++pe) st_cluster_v4(mapa_cluster(off, static_cast<uint32_t>(pe)), v);
  };
  // per-row (mean, M2) of this CTA's y slice -> every CTA's s_st[rank]
  auto ln_stats = [&]() {
    const int r = tid >> 3, sub = tid & 7;                  // 8 threads per row
    if (r < ROWS) {
      float v[DS / 8];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < DS / 8; ++i) { v[i] = s_y[r * DS + sub + 8 * i]; s += v[i]; }
      s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2); s += __shfl_xor_sync(0xffffffffu, s, 4);
      const float mean = s * (1.0f / DS);
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < DS / 8; ++i) { const float d = v[i] - mean; q += d * d; }
      q += __shfl_xor_sync(0xffffffffu, q, 1); q += __shfl_xor_sync(0xffffffffu, q, 2); q += __shfl_xor_sync(0xffffffffu, q, 4);
      // lane `sub` of the row group delivers to peer `sub`
      if (sub < CS) st_cluster_v2f(mapa_cluster(smem_u32(&s_st[rank * ROWS + r]), static_cast<uint32_t>(sub)), mean, q);
    }
  };
  // merge the 8 slice statistics (fixed order: identical in every CTA), normalise this CTA's slice, all-gather bf16
  auto ln_apply = [&](const float* __restrict__ gamma, const float* __restrict__ beta, uint8_t* abuf) {
    if (tid < ROWS) {
      float n = 0.f, mean = 0.f, m2 = 0.f;
#pragma unroll
      for (int k = 0; k < CS; ++k) {
        const float2 s = s_st[k * ROWS + tid];
        const float nb = static_cast<float>(DS), nn = n + nb;
        const float delta = s.x - mean;
        mean += delta * (nb / nn);
        m2 += s.y + delta * delta * (n * nb / nn);
        n = nn;
      }
      s_mr[tid] = make_float2(mean, 1.0f / sqrtf(m2 * (1.0f / D) + 1e-5f));
    }
    a2_csync();
    for (int i = tid; i < ROWS * (DS / 8); i += A2_THREADS) {
      const int r = i / (DS / 8), ch = i % (DS / 8);
      const float2 mr = s_mr[r];
      const int c0 = rank * DS + ch * 8;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        o[j] = (s_y[r * DS + ch * 8 + j] - mr.x) * mr.y * __ldg(gamma + c0 + j) + __ldg(beta + c0 + j);
      bcast16(abuf, r, c0, make_uint4(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]), pack_bf16(o[4], o[5]), pack_bf16(o[6], o[7])));
    }
  };
  // D x D projection of this CTA's column slice: acc = A[ROWS, D] * Wslice[DS, D]^T  (consumes NSL_S ring slots)
  constexpr int NT_S = DS / 8;                                   // n8 tiles of the slice
  constexpr int NTW_S = (((NT_S + G - 1) / G) + 1) & ~1;         // per warp, even
  auto gemm_slice = [&](const uint8_t* abuf, float (&acc)[NTW_S][4]) {
#pragma unroll
    for (int j = 0; j < NTW_S; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int sl = 0; sl < Cfg::NSL_S; ++sl) {
      const uint8_t* slot = ring.wait();
      const int k0 = sl * Cfg::GS;
      const int n = (KT - k0 < Cfg::GS) ? (KT - k0) : Cfg::GS;
      for (int i = 0; i < n; ++i) mma_box<NTW_S>(acc, abuf + (k0 + i) * ROWS * 128, mi, slot + i * DS * 128, ng * NTW_S, lane);
      ring.release();
    }
  };

#define A2_PROF4(slot)                                                                                          \
  do {                                                                                                          \
    if (p.prof != nullptr && blockIdx.x == 0 && tid == 0 && step == 1) p.prof[26 * 16 + (slot)] = a2_timer_ns(); \
  } while (0)
  // the [32][16] profile buffer: rows 0..25 are steps, row 26 the extra stamps of step 1 (A2_PROF4); the 64-pitch
  // kernels (L > 32) record steps < 26 only
#define A2_PROF(slot)                                                                                           \
  do {                                                                                                          \
    if (p.prof != nullptr && blockIdx.x == 0 && tid == 0 && (IDP == 32 || step < A2_PROF_STEPS))                \
      p.prof[step * 16 + (slot)] = a2_timer_ns();                                                               \
  } while (0)

  for (int step = 0; step < p.L; ++step) {
    const int nkeys = step + 1;
    A2_PROF(0);
    // ================= P1: self-attention over the (position, token) table: thread = (own row, 8-dim chunk) =================
    {
      const int items = n_own * (D / 8);
      for (int base = 0; base < items; base += A2_THREADS) {        // warp-uniform trip count
        if (base + warp * 32 >= items) break;                        // whole warp idle (warp-uniform)
        const int it = base + tid;
        const bool valid = it < items;
        const int itc = valid ? it : items - 1;
        const int oi = itc / (D / 8), ch = itc % (D / 8);
        const int r = rank + CS * oi;
        const int* idr = s_ids + r * IDP;
        float q[8];
        {
          const float4 q0 = __ldg(reinterpret_cast<const float4*>(p.qs + static_cast<long long>(step) * D + ch * 8));
          const float4 q1 = __ldg(reinterpret_cast<const float4*>(p.qs + static_cast<long long>(step) * D + ch * 8 + 4));
          q[0] = q0.x; q[1] = q0.y; q[2] = q0.z; q[3] = q0.w; q[4] = q1.x; q[5] = q1.y; q[6] = q1.z; q[7] = q1.w;
        }
        float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int j0 = 0; j0 < nkeys; j0 += 8) {
          uint4 kk[8], vv[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int j = (j0 + u < nkeys) ? (j0 + u) : (nkeys - 1);
            const __nv_bfloat16* row = p.kvtab + (static_cast<long long>(j) * p.V + idr[j]) * (2 * D) + ch * 8;
            kk[u] = __ldg(reinterpret_cast<const uint4*>(row));
            vv[u] = __ldg(reinterpret_cast<const uint4*>(row + D));
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            if (j0 + u < nkeys) {                                      // uniform over the CTA
              const __nv_bfloat162* k2 = reinterpret_cast<const __nv_bfloat162*>(&kk[u]);
              float s = 0.f;
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(k2[e]);
                s = fmaf(q[2 * e], f.x, s);
                s = fmaf(q[2 * e + 1], f.y, s);
              }
              s += __shfl_xor_sync(0xffffffffu, s, 1);                 // 4 consecutive chunks = one 32-dim head
              s += __shfl_xor_sync(0xffffffffu, s, 2);
              const float mn = fmaxf(m, s);
              const float sc = expf(m - mn), pj = expf(s - mn);
              l = l * sc + pj;
              const __nv_bfloat162* v2 = reinterpret_cast<const __nv_bfloat162*>(&vv[u]);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(v2[e]);
                acc[2 * e] = fmaf(acc[2 * e], sc, pj * f.x);
                acc[2 * e + 1] = fmaf(acc[2 * e + 1], sc, pj * f.y);
              }
              m = mn;
            }
          }
        }
        if (valid) {
          const float inv = 1.0f / l;
          bcast16(s_a2, r, ch * 8,
                  make_uint4(pack_bf16(acc[0] * inv, acc[1] * inv), pack_bf16(acc[2] * inv, acc[3] * inv),
                             pack_bf16(acc[4] * inv, acc[5] * inv), pack_bf16(acc[6] * inv, acc[7] * inv)));
        }
      }
    }
    A2_PROF(1);
    cluster_sync_relacq();                                                                            // (1) sa gathered
    A2_PROF(2);
    // ================= P2: y = pos_queries[step] + out_proj(sa) (this CTA's columns) =================
    {
      float acc[NTW_S][4];
      gemm_slice(s_a2, acc);
#pragma unroll
      for (int j = 0; j < NTW_S; ++j) {
        const int nt = ng * NTW_S + j;
        if (nt < NT_S) {
          const int c = nt * 8 + 2 * t, cg = rank * DS + c;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bo_s + cg));
          const float2 pq2 = __ldg(reinterpret_cast<const float2*>(p.posq + static_cast<long long>(step) * D + cg));
          const int r0 = mi * 16 + g;
          *reinterpret_cast<float2*>(&s_y[r0 * DS + c]) = make_float2(acc[j][0] + bb.x + pq2.x, acc[j][1] + bb.y + pq2.y);
          *reinterpret_cast<float2*>(&s_y[(r0 + 8) * DS + c]) = make_float2(acc[j][2] + bb.x + pq2.x, acc[j][3] + bb.y + pq2.y);
        }
      }
      a2_csync();
      ln_stats();
    }
    A2_PROF(3);
    cluster_sync_relacq();                                                                            // (2) LN1 statistics
    ln_apply(p.g1, p.be1, s_a1);
    A2_PROF(4);
    cluster_sync_relacq();                                                                            // (3) LN1(y) gathered
    // ================= P3: qc = scale * q_proj(LN1(y)); each row goes to the CTA that owns it =================
    {
      float acc[NTW_S][4];
      gemm_slice(s_a1, acc);
#pragma unroll
      for (int j = 0; j < NTW_S; ++j) {
        const int nt = ng * NTW_S + j;
        if (nt < NT_S) {
          const int cg = rank * DS + nt * 8 + 2 * t;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bq_c + cg));
          const int r0 = mi * 16 + g, r1 = r0 + 8;
          if (hs) {                      // the 64-column block goes to the CTA that owns (row, k-block)
            if (r0 < nrows)
              st_cluster_v2f(mapa_cluster(smem_u32(&s_q[cg]), static_cast<uint32_t>(r0 * KT + (cg >> 6))),
                             (acc[j][0] + bb.x) * p.qscale, (acc[j][1] + bb.y) * p.qscale);
            if (r1 < nrows)
              st_cluster_v2f(mapa_cluster(smem_u32(&s_q[cg]), static_cast<uint32_t>(r1 * KT + (cg >> 6))),
                             (acc[j][2] + bb.x) * p.qscale, (acc[j][3] + bb.y) * p.qscale);
          } else {
            st_cluster_v2f(mapa_cluster(smem_u32(&s_q[(r0 / CS) * D + cg]), static_cast<uint32_t>(r0 % CS)),
                           (acc[j][0] + bb.x) * p.qscale, (acc[j][1] + bb.y) * p.qscale);
            st_cluster_v2f(mapa_cluster(smem_u32(&s_q[(r1 / CS) * D + cg]), static_cast<uint32_t>(r1 % CS)),
                           (acc[j][2] + bb.x) * p.qscale, (acc[j][3] + bb.y) * p.qscale);
          }
        }
      }
    }
    A2_PROF(5);
    cluster_sync_relacq();                                                                            // (4) queries delivered
    A2_PROF(6);
    // ================= P4: cross-attention of the owned images; K/V stream through the ring =================
    {
      const int ntk = p.tbox >> 6;                    // n8 tiles of keys per warp inside a key block (tbox / 8 warps / 8)
      const int kw = ntk * 8;                         // keys per warp per block
      A2_PROF4(0);
      const int kb_lo = hs ? hs_kb : 0, kb_hi = hs ? hs_kb + 1 : KT;      // k-blocks (head pairs) this CTA computes per pass
      for (int oi = 0; oi < c_own; ++oi) {
        const int r = hs ? hs_row : rank + CS * oi;
        const float* qrow = s_q + oi * D;
        // the query's A-operand words, split into bf16 hi + lo (q = hi + lo to ~16 mantissa bits), once per image
        for (int i = kb_lo * 16 + tid; i < kb_hi * 16; i += A2_THREADS) {
          const float* qd = qrow + (i >> 2) * 16 + 2 * (i & 3);        // (kb, ks) = i / 4, thread-in-quad t = i % 4
          const float q0 = qd[0], q1 = qd[1], q8 = qd[8], q9 = qd[9];
          const float h0 = __bfloat162float(__float2bfloat16_rn(q0)), h1 = __bfloat162float(__float2bfloat16_rn(q1));
          const float h8 = __bfloat162float(__float2bfloat16_rn(q8)), h9 = __bfloat162float(__float2bfloat16_rn(q9));
          s_qf[i] = make_uint4(pack_bf16(h0, h1), pack_bf16(h8, h9), pack_bf16(q0 - h0, q1 - h1), pack_bf16(q8 - h8, q9 - h9));
        }
        a2_csync();
        float sacc[MH][2][2][4];                      // [m tile][key block][n8 tile][frag]; q_hi term
        float slo[MH][2][2][4];                       // q_lo term: its own dependency chain, added before the softmax
#pragma unroll
        for (int a = 0; a < MH; ++a)
#pragma unroll
          for (int b = 0; b < 2; ++b)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              sacc[a][b][c][0] = sacc[a][b][c][1] = sacc[a][b][c][2] = sacc[a][b][c][3] = 0.f;
              slo[a][b][c][0] = slo[a][b][c][1] = slo[a][b][c][2] = slo[a][b][c][3] = 0.f;
            }
        // ---- S = Q_blockdiag K^T: K box kb holds dims [64 kb, 64 kb + 64) = heads 2 kb, 2 kb + 1 ----
        for (int kb = kb_lo; kb < kb_hi; ++kb) {
#pragma unroll
          for (int tbi = 0; tbi < 2; ++tbi) {
            if (tbi < p.tb) {
              const uint8_t* box = ring.wait();
              const uint32_t bbase = smem_u32(box);
              const int mh = (2 * kb) / 16;
#pragma unroll
              for (int ks = 0; ks < 4; ++ks) {
                const int hrow = (2 * kb + (ks >> 1)) & 15;           // row of this k-step's head inside its m tile
                const uint4 qf = s_qf[(kb * 4 + ks) * 4 + t];
                const uint32_t hi01 = qf.x, hi89 = qf.y, lo01 = qf.z, lo89 = qf.w;
                const bool top = (g == hrow), bot = (g + 8 == hrow);
                const uint32_t ah0 = top ? hi01 : 0u, ah1 = bot ? hi01 : 0u, ah2 = top ? hi89 : 0u, ah3 = bot ? hi89 : 0u;
                const uint32_t al0 = top ? lo01 : 0u, al1 = bot ? lo01 : 0u, al2 = top ? lo89 : 0u, al3 = bot ? lo89 : 0u;
                const int n = warp * kw + (lane & 7) + (lane >> 4) * 8;
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(bbase + box_off(n, ks * 16 + ((lane >> 3) & 1) * 8), b0, b1, b2, b3);
#pragma unroll
                for (int a = 0; a < MH; ++a) {
                  if (a == mh) {
                    mma_bf16_16816(sacc[a][tbi][0], ah0, ah1, ah2, ah3, b0, b1);
                    mma_bf16_16816(slo[a][tbi][0], al0, al1, al2, al3, b0, b1);
                    if (ntk == 2) {
                      mma_bf16_16816(sacc[a][tbi][1], ah0, ah1, ah2, ah3, b2, b3);
                      mma_bf16_16816(slo[a][tbi][1], al0, al1, al2, al3, b2, b3);
                    }
                  }
                }
              }
              ring.release();
            }
          }
        }
        if (oi < 4) A2_PROF4(1 + 3 * oi);
        // ---- softmax over the keys (rows = heads): mask, the 8 warps reduce through shared memory ----
        float rmax[MH][2];
#pragma unroll
        for (int a = 0; a < MH; ++a) {
#pragma unroll
          for (int tbi = 0; tbi < 2; ++tbi)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
              for (int f = 0; f < 4; ++f) sacc[a][tbi][c][f] += slo[a][tbi][c][f];
          rmax[a][0] = rmax[a][1] = -INFINITY;
#pragma unroll
          for (int tbi = 0; tbi < 2; ++tbi)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int key = tbi * 128 + warp * kw + c * 8 + 2 * t;
              const bool live = (tbi < p.tb) && (c < ntk);
              if (!live || key >= p.T) { sacc[a][tbi][c][0] = -INFINITY; sacc[a][tbi][c][2] = -INFINITY; }
              if (!live || key + 1 >= p.T) { sacc[a][tbi][c][1] = -INFINITY; sacc[a][tbi][c][3] = -INFINITY; }
              rmax[a][0] = fmaxf(rmax[a][0], fmaxf(sacc[a][tbi][c][0], sacc[a][tbi][c][1]));
              rmax[a][1] = fmaxf(rmax[a][1], fmaxf(sacc[a][tbi][c][2], sacc[a][tbi][c][3]));
            }
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            rmax[a][hf] = fmaxf(rmax[a][hf], __shfl_xor_sync(0xffffffffu, rmax[a][hf], 1));
            rmax[a][hf] = fmaxf(rmax[a][hf], __shfl_xor_sync(0xffffffffu, rmax[a][hf], 2));
          }
          if (t == 0) {
            s_red[warp * (MH * 16) + a * 16 + g] = rmax[a][0];
            s_red[warp * (MH * 16) + a * 16 + g + 8] = rmax[a][1];
          }
        }
        a2_csync();
        float rsum[MH][2];
#pragma unroll
        for (int a = 0; a < MH; ++a) {
          float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            m0 = fmaxf(m0, s_red[w * (MH * 16) + a * 16 + g]);
            m1 = fmaxf(m1, s_red[w * (MH * 16) + a * 16 + g + 8]);
          }
          rsum[a][0] = rsum[a][1] = 0.f;
#pragma unroll
          for (int tbi = 0; tbi < 2; ++tbi)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              if (tbi < p.tb && c < ntk) {
                const float e0 = expf(sacc[a][tbi][c][0] - m0), e1 = expf(sacc[a][tbi][c][1] - m0);
                const float e2 = expf(sacc[a][tbi][c][2] - m1), e3 = expf(sacc[a][tbi][c][3] - m1);
                rsum[a][0] += e0 + e1;
                rsum[a][1] += e2 + e3;
                // P (hi, lo) -> A-operand tiles [16 MH rows][256 keys]: tile = key / 64
                const int key = tbi * 128 + warp * kw + c * 8 + 2 * t;
                const __nv_bfloat16 f0 = __float2bfloat16_rn(e0), f1 = __float2bfloat16_rn(e1), f2 = __float2bfloat16_rn(e2),
                                    f3 = __float2bfloat16_rn(e3);
                const uint32_t off0 = a_off<MH * 16>(a * 16 + g, key), off1 = a_off<MH * 16>(a * 16 + g + 8, key);
                *reinterpret_cast<uint32_t*>(s_p + off0) = pack_bf16(__bfloat162float(f0), __bfloat162float(f1));
                *reinterpret_cast<uint32_t*>(s_p + off1) = pack_bf16(__bfloat162float(f2), __bfloat162float(f3));
                *reinterpret_cast<uint32_t*>(s_p + Cfg::P_BYTES / 2 + off0) =
                    pack_bf16(e0 - __bfloat162float(f0), e1 - __bfloat162float(f1));
                *reinterpret_cast<uint32_t*>(s_p + Cfg::P_BYTES / 2 + off1) =
                    pack_bf16(e2 - __bfloat162float(f2), e3 - __bfloat162float(f3));
              }
            }
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            rsum[a][hf] += __shfl_xor_sync(0xffffffffu, rsum[a][hf], 1);
            rsum[a][hf] += __shfl_xor_sync(0xffffffffu, rsum[a][hf], 2);
          }
          if (t == 0) {
            s_red[8 * MH * 16 + warp * (MH * 16) + a * 16 + g] = rsum[a][0];
            s_red[8 * MH * 16 + warp * (MH * 16) + a * 16 + g + 8] = rsum[a][1];
          }
        }
        a2_csync();
        if (oi < 4) A2_PROF4(2 + 3 * oi);
        // ---- O = P V, split over the KEYS: warp w owns the k16 step w of every key block, so its P fragments (hi + lo)
        // are loaded once per image and every V box is read from shared memory exactly once (a split over the dims re-read
        // the whole P tile in every warp for every box: 4x the box's own bytes).  Per box: 64 dims = 8 n8 tiles; the two
        // heads' rows of the 16 x 64 partial product go to s_part[warp], summed over the warps after the last box.
        {
          const int nsteps = p.tbox >> 4;                      // k16 steps per key block (4 or 8)
          const bool has_step = warp < nsteps;
          const int prow = (lane & 7) + ((lane >> 3) & 1) * 8;
          uint32_t ph[2][4], pl[2][4];                         // [key block][frag]
          int cur_mh = -1;
          for (int kb = kb_lo; kb < kb_hi; ++kb) {
            const int mh = (2 * kb) >> 4;
            if (mh != cur_mh) {                                // (re)load this warp's P fragments for the m16 tile of heads
              cur_mh = mh;
#pragma unroll
              for (int tbi = 0; tbi < 2; ++tbi) {
                if (tbi < p.tb && has_step) {
                  const uint32_t pa = smem_u32(s_p) + a_off<MH * 16>(mh * 16 + prow, tbi * 128 + warp * 16 + (lane >> 4) * 8);
                  ldmatrix_x4(pa, ph[tbi][0], ph[tbi][1], ph[tbi][2], ph[tbi][3]);
                  ldmatrix_x4(pa + Cfg::P_BYTES / 2, pl[tbi][0], pl[tbi][1], pl[tbi][2], pl[tbi][3]);
                }
              }
            }
            float oacc[8][4];
#pragma unroll
            for (int j = 0; j < 8; ++j) oacc[j][0] = oacc[j][1] = oacc[j][2] = oacc[j][3] = 0.f;
#pragma unroll
            for (int tbi = 0; tbi < 2; ++tbi) {
              if (tbi < p.tb) {
                const uint8_t* box = ring.wait();
                if (has_step) {
                  const int vr = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;      // key row of this lane's 8x8 matrix
                  const uint32_t vb = smem_u32(box) + static_cast<uint32_t>(vr * 128);
                  const uint32_t vx = static_cast<uint32_t>(vr & 7);
#pragma unroll
                  for (int np = 0; np < 4; ++np) {                                     // dims 16 np .. 16 np + 15 of the box
                    uint32_t v0, v1, v2, v3;
                    ldmatrix_x4_trans(vb + (((static_cast<uint32_t>(np * 2) + (lane >> 4)) ^ vx) << 4), v0, v1, v2, v3);
                    mma_bf16_16816(oacc[2 * np], ph[tbi][0], ph[tbi][1], ph[tbi][2], ph[tbi][3], v0, v1);
                    mma_bf16_16816(oacc[2 * np + 1], ph[tbi][0], ph[tbi][1], ph[tbi][2], ph[tbi][3], v2, v3);
                    mma_bf16_16816(oacc[2 * np], pl[tbi][0], pl[tbi][1], pl[tbi][2], pl[tbi][3], v0, v1);
                    mma_bf16_16816(oacc[2 * np + 1], pl[tbi][0], pl[tbi][1], pl[tbi][2], pl[tbi][3], v2, v3);
                  }
                }
                ring.release();
              }
            }
            // rows of the two heads of this box: n8 tiles 0..3 -> head 2 kb, tiles 4..7 -> head 2 kb + 1
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int hr = (2 * kb + (j >> 2)) & 15;
              if ((hr & 7) == g) {
                const float2 v = (hr < 8) ? make_float2(oacc[j][0], oacc[j][1]) : make_float2(oacc[j][2], oacc[j][3]);
                *reinterpret_cast<float2*>(&s_part[warp * D + kb * 64 + j * 8 + 2 * t]) = has_step ? v : make_float2(0.f, 0.f);
              }
            }
          }
          a2_csync();
          // sum the 8 key slices (fixed order), normalise by the row sum of the head, round to bf16
          for (int i = kb_lo * 32 + tid; i < kb_hi * 32; i += A2_THREADS) {
            const int d0 = 2 * i, hh = d0 >> 5;
            float tot = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) tot += s_red[8 * MH * 16 + w * (MH * 16) + hh];
            float2 o = *reinterpret_cast<const float2*>(&s_part[d0]);
#pragma unroll
            for (int w = 1; w < 8; ++w) {
              const float2 q2 = *reinterpret_cast<const float2*>(&s_part[w * D + d0]);
              o.x += q2.x; o.y += q2.y;
            }
            const float inv = 1.0f / tot;
            *reinterpret_cast<uint32_t*>(&s_ca[d0]) = pack_bf16(o.x * inv, o.y * inv);
          }
        }
        a2_csync();
        for (int ch = kb_lo * 8 + tid; ch < kb_hi * 8; ch += A2_THREADS)
          bcast16(s_a2, r, ch * 8, *reinterpret_cast<const uint4*>(&s_ca[ch * 8]));
        if (oi < 4) A2_PROF4(3 + 3 * oi);
      }
    }
    A2_PROF(7);
    cluster_sync_relacq();                                                                            // (5) ca gathered
    A2_PROF(8);
    // ================= P5: y += out_proj(ca) =================
    {
      float acc[NTW_S][4];
      gemm_slice(s_a2, acc);
#pragma unroll
      for (int j = 0; j < NTW_S; ++j) {
        const int nt = ng * NTW_S + j;
        if (nt < NT_S) {
          const int c = nt * 8 + 2 * t, cg = rank * DS + c;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bo_c + cg));
          const int r0 = mi * 16 + g;
          float2* d0 = reinterpret_cast<float2*>(&s_y[r0 * DS + c]);
          float2* d1 = reinterpret_cast<float2*>(&s_y[(r0 + 8) * DS + c]);
          const float2 o0 = *d0, o1 = *d1;
          *d0 = make_float2(o0.x + (acc[j][0] + bb.x), o0.y + (acc[j][1] + bb.y));
          *d1 = make_float2(o1.x + (acc[j][2] + bb.x), o1.y + (acc[j][3] + bb.y));
        }
      }
      a2_csync();
      ln_stats();
    }
    A2_PROF(9);
    cluster_sync_relacq();                                                                            // (6) LN2 statistics
    ln_apply(p.g2, p.be2, s_a1);
    cluster_sync_relacq();                                                                            // (7) LN2(y) gathered
    A2_PROF(10);
    // ================= P6: hd = GELU(linear1(LN2(y))) for this CTA's hidden slice (stays local) =================
    {
      constexpr int NT1 = Cfg::NC1 / 8;
      constexpr int NTW1 = (((NT1 + G - 1) / G) + 1) & ~1;
      for (int c = 0; c < Cfg::NCH1; ++c) {
        float acc[NTW1][4];
#pragma unroll
        for (int j = 0; j < NTW1; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        for (int kb = 0; kb < KT; ++kb) {
          const uint8_t* slot = ring.wait();
          mma_box<NTW1>(acc, s_a1 + kb * ROWS * 128, mi, slot, ng * NTW1, lane);
          ring.release();
        }
#pragma unroll
        for (int j = 0; j < NTW1; ++j) {
          const int nt = ng * NTW1 + j;
          if (nt < NT1) {
            const int cl_ = c * Cfg::NC1 + nt * 8 + 2 * t;              // column inside the hidden slice
            const float2 bb = __ldg(reinterpret_cast<const float2*>(p.b1 + rank * MS + cl_));
            const int r0 = mi * 16 + g;
            *reinterpret_cast<uint32_t*>(s_hd + a_off<ROWS>(r0, cl_)) = pack_bf16(gelu_erf(acc[j][0] + bb.x), gelu_erf(acc[j][1] + bb.y));
            *reinterpret_cast<uint32_t*>(s_hd + a_off<ROWS>(r0 + 8, cl_)) = pack_bf16(gelu_erf(acc[j][2] + bb.x), gelu_erf(acc[j][3] + bb.y));
          }
        }
      }
      a2_csync();
    }
    A2_PROF(11);
    // ================= P7: partial linear2 over this CTA's K slice -> column owners =================
    {
      constexpr int NT2 = Cfg::NC2 / 8;
      constexpr int NTW2 = (((NT2 + G - 1) / G) + 1) & ~1;
      for (int c = 0; c < Cfg::NCH2; ++c) {
        float acc[NTW2][4];
#pragma unroll
        for (int j = 0; j < NTW2; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        for (int kb = 0; kb < KT2; ++kb) {
          const uint8_t* slot = ring.wait();
          const int ksteps = (MS - kb * 64 >= 64) ? 4 : ((MS - kb * 64) / 16);
          mma_box<NTW2>(acc, s_hd + kb * ROWS * 128, mi, slot, ng * NTW2, lane, ksteps);
          ring.release();
        }
#pragma unroll
        for (int j = 0; j < NTW2; ++j) {
          const int nt = ng * NTW2 + j;
          if (nt < NT2) {
            const int cg = c * Cfg::NC2 + nt * 8 + 2 * t;               // global output column
            const int dst = cg / DS, cc = cg % DS;
            const int r0 = mi * 16 + g;
            st_cluster_v2f(mapa_cluster(smem_u32(&s_recv[(rank * ROWS + r0) * DS + cc]), static_cast<uint32_t>(dst)), acc[j][0], acc[j][1]);
            st_cluster_v2f(mapa_cluster(smem_u32(&s_recv[(rank * ROWS + r0 + 8) * DS + cc]), static_cast<uint32_t>(dst)), acc[j][2], acc[j][3]);
          }
        }
      }
    }
    A2_PROF(12);
    cluster_sync_relacq();                                                                            // (8) partials delivered
    // ================= y += b2 + sum of the 8 partials (fixed order) =================
    for (int i = tid; i < ROWS * DS; i += A2_THREADS) {
      const int c = i % DS;
      float s = s_recv[i];
#pragma unroll
      for (int k = 1; k < CS; ++k) s += s_recv[k * ROWS * DS + i];
      s_y[i] += s + __ldg(p.b2 + rank * DS + c);
    }
    a2_csync();
    ln_stats();
    A2_PROF(13);
    cluster_sync_relacq();                                                                            // (9) LN3 statistics
    ln_apply(p.g3, p.be3, s_a1);
    cluster_sync_relacq();                                                                            // (10) LN3(y) gathered
    A2_PROF(14);
    // ================= P8: logits[:, step] = head(LN3(y)) in every CTA; greedy token =================
    if constexpr (WIDE) {
      // class slice [c_lo, c_hi) of this CTA, 128 classes per chunk; every chunk multiplies all rows in the k order of
      // mma_box; logits leave from the fragments; a running (max, lowest index) per (thread, row)
      constexpr int NTH = 16;                                           // 128 columns
      constexpr int NTWH = (((NTH + G - 1) / G) + 1) & ~1;
      const int c_lo = rank * h_cs;
      const int c_hi = (c_lo + h_cs < p.C) ? (c_lo + h_cs) : p.C;
      const int r0 = mi * 16 + g;
      float* lrow0 = p.logits + (static_cast<long long>(img0 + r0) * p.L + step) * p.C;
      float* lrow1 = p.logits + (static_cast<long long>(img0 + r0 + 8) * p.L + step) * p.C;
      const bool st0 = r0 < nrows, st1 = r0 + 8 < nrows;
      // allowlist words of the two rows, read through L2 per column (a row is up to 512 words: not staged)
      const uint32_t* mrow0 = (p.mask != nullptr && st0) ? p.mask + (img0 + r0) * class_mask_words(p.C) : nullptr;
      const uint32_t* mrow1 = (p.mask != nullptr && st1) ? p.mask + (img0 + r0 + 8) * class_mask_words(p.C) : nullptr;
      float best0 = -INFINITY, best1 = -INFINITY;
      int bi0 = ARGMAX_NONE, bi1 = ARGMAX_NONE;
      for (int hc = 0; hc < h_chunks; ++hc) {
        float acc[NTWH][4];
#pragma unroll
        for (int j = 0; j < NTWH; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
        for (int kb = 0; kb < KT; ++kb) {
          const uint8_t* slot = ring.wait();
          mma_box<NTWH>(acc, s_a1 + kb * ROWS * 128, mi, slot, ng * NTWH, lane);
          ring.release();
        }
#pragma unroll
        for (int j = 0; j < NTWH; ++j) {
          const int nt = ng * NTWH + j;
          if (nt < NTH) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {                               // columns in increasing order per thread
              const int c = c_lo + hc * 128 + nt * 8 + 2 * t + e;
              if (c < c_hi) {
                const float b = __ldg(p.bh + c);
                float v0 = acc[j][e] + b, v1 = acc[j][2 + e] + b;
                if (mrow0 != nullptr && !class_allowed(mrow0, c)) v0 = -INFINITY;
                if (mrow1 != nullptr && !class_allowed(mrow1, c)) v1 = -INFINITY;
                if (st0) lrow0[c] = v0;
                if (st1) lrow1[c] = v1;
                argmax_fold(best0, bi0, v0, c);
                argmax_fold(best1, bi1, v1, c);
              }
            }
          }
        }
      }
      // quad (same rows, interleaved columns), then the G warps of the m16 tile, in torch.argmax order (ptx.cuh)
      argmax_shfl(best0, bi0, 1, 4);
      argmax_shfl(best1, bi1, 1, 4);
      float* s_hv = s_log;                                              // [ROWS][G] warp maxima (P is dead here)
      int* s_hi = reinterpret_cast<int*>(s_log + ROWS * G);
      if (t == 0) {
        s_hv[r0 * G + ng] = best0; s_hi[r0 * G + ng] = bi0;
        s_hv[(r0 + 8) * G + ng] = best1; s_hi[(r0 + 8) * G + ng] = bi1;
      }
      a2_csync();
      // this CTA's pair of row r -> s_st[rank][r] of every CTA (s_st is free: the LN3 statistics were read before (10))
      if (tid < ROWS) {
        float bv = s_hv[tid * G];
        int bx = s_hi[tid * G];
#pragma unroll
        for (int w = 1; w < G; ++w) argmax_fold(bv, bx, s_hv[tid * G + w], s_hi[tid * G + w]);
        const uint32_t off = smem_u32(&s_st[rank * ROWS + tid]);
#pragma unroll
        for (int pe = 0; pe < CS; ++pe) st_cluster_v2f(mapa_cluster(off, static_cast<uint32_t>(pe)), bv, __int_as_float(bx));
      }
      cluster_sync_relacq();                                                                          // (11) pairs exchanged
      // every CTA folds the same CS pairs in rank order under the same total order: the same token in every CTA, the
      // one torch.argmax picks (an empty tail slice sends ARGMAX_NONE, which never wins)
      if (tid < nrows) {
        const int r = tid;
        const long long b = img0 + r;
        float bv = s_st[r].x;
        int bx = __float_as_int(s_st[r].y);
#pragma unroll
        for (int k = 1; k < CS; ++k) {
          const float2 s = s_st[k * ROWS + r];
          argmax_fold(bv, bx, s.x, __float_as_int(s.y));
        }
        if (step + 1 < p.L) {
          int v = bx;
          if (p.forced != nullptr) v = p.forced[b * p.forced_ld + step + 1];
          s_ids[r * IDP + step + 1] = v;
          if ((r % CS) == rank) p.ids[b * p.ids_ld + step + 1] = v;     // one CTA stores the row
        }
      }
      a2_csync();
    } else {
      constexpr int NTH = 12;                                           // 96 columns
      constexpr int NTWH = (((NTH + G - 1) / G) + 1) & ~1;
      float acc[NTWH][4];
#pragma unroll
      for (int j = 0; j < NTWH; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
      for (int kb = 0; kb < KT; ++kb) {
        const uint8_t* slot = ring.wait();
        mma_box<NTWH>(acc, s_a1 + kb * ROWS * 128, mi, slot, ng * NTWH, lane);
        ring.release();
      }
#pragma unroll
      for (int j = 0; j < NTWH; ++j) {
        const int nt = ng * NTWH + j;
        if (nt < NTH) {
          const int c = nt * 8 + 2 * t;
          const float b0 = (c < p.C) ? __ldg(p.bh + c) : 0.f, b1 = (c + 1 < p.C) ? __ldg(p.bh + c + 1) : 0.f;
          const int r0 = mi * 16 + g;
          s_log[r0 * A2_SLOG_LD + c] = acc[j][0] + b0;
          s_log[r0 * A2_SLOG_LD + c + 1] = acc[j][1] + b1;
          s_log[(r0 + 8) * A2_SLOG_LD + c] = acc[j][2] + b0;
          s_log[(r0 + 8) * A2_SLOG_LD + c + 1] = acc[j][3] + b1;
        }
      }
      a2_csync();
      if (p.mask != nullptr) {
        // allowlist: the same (warp, lane) -> (row, column) map as the store / argmax loop below, so no barrier between
        for (int r = warp; r < nrows; r += 8) {
          const uint32_t* mrow = p.mask + (img0 + r) * class_mask_words(p.C);
          for (int j = lane; j < p.C; j += 32)
            if (!class_allowed(mrow, j)) s_log[r * A2_SLOG_LD + j] = -INFINITY;
        }
      }
      for (int r = warp; r < nrows; r += 8) {
        const long long b = img0 + r;
        float* lrow = p.logits + (b * p.L + step) * p.C;
        const bool writer = (r % CS) == rank;                        // one CTA stores the row
        float best = -INFINITY;
        int bi = ARGMAX_NONE;
        for (int j = lane; j < p.C; j += 32) {
          const float v = s_log[r * A2_SLOG_LD + j];
          if (writer) lrow[j] = v;
          argmax_scan(best, bi, v, j);
        }
        bi = argmax_finish(best, bi, s_log + r * A2_SLOG_LD, p.C, lane);
        if (lane == 0 && step + 1 < p.L) {
          int v = bi;
          if (p.forced != nullptr) v = p.forced[b * p.forced_ld + step + 1];
          s_ids[r * IDP + step + 1] = v;
          if (writer) p.ids[b * p.ids_ld + step + 1] = v;
        }
      }
      a2_csync();
    }
    A2_PROF(15);
  }
#undef A2_PROF
#undef A2_PROF4
  }
  cluster_sync_relacq();       // no CTA exits while a peer may still address its shared memory
}

template <int D, int MT, int CS, bool HS = false>
__global__ void __launch_bounds__(A2_LAUNCH_THREADS, 1)
dec_ar2_kernel(const __grid_constant__ DecAr2Maps maps, const DecAr2Params p) {
  dec_ar2_body<D, MT, CS, HS, false, 32>(maps, p);
}
template <int D, int MT, int CS, bool HS = false>
__global__ void __launch_bounds__(A2_LAUNCH_THREADS, 1)
dec_ar2_wide_kernel(const __grid_constant__ DecAr2Maps maps, const DecAr2Params p) {
  dec_ar2_body<D, MT, CS, HS, true, 32>(maps, p);
}
// labels of 32..63 characters (33..64 decode positions): ids rows of 64 in shared memory and in p.ids
template <int D, int MT, int CS, bool HS = false>
__global__ void __launch_bounds__(A2_LAUNCH_THREADS, 1)
dec_ar2_long_kernel(const __grid_constant__ DecAr2Maps maps, const DecAr2Params p) {
  dec_ar2_body<D, MT, CS, HS, false, 64>(maps, p);
}
template <int D, int MT, int CS, bool HS = false>
__global__ void __launch_bounds__(A2_LAUNCH_THREADS, 1)
dec_ar2_long_wide_kernel(const __grid_constant__ DecAr2Maps maps, const DecAr2Params p) {
  dec_ar2_body<D, MT, CS, HS, true, 64>(maps, p);
}

// ------------------------------------------------------------------------------------------------------------------
// Microbenchmark (tests/bench_tma_stream.py): the ring protocol of the AR kernel with no compute - every CTA streams
// `nboxes` [128 x 64] bf16 boxes (16 KB) of a column-blocked buffer through `nslot` slots.  Launched with different
// cluster sizes to measure what a CTA can ingest through TMA inside a cluster.
__global__ void __launch_bounds__(A2_THREADS + 32, 1)
tma_stream_bench_kernel(const __grid_constant__ CUtensorMap map, int nboxes, int nslot, int row_boxes, int blocks, int mode,
                        unsigned int* sink) {
  // mode bit 0: every thread polls the full barrier (else one lane per warp); bit 1: a dedicated producer warp (warp 8)
  // refills slots behind per-slot empty barriers, the 8 consumer warps never meet at a CTA barrier
  extern __shared__ uint8_t bs_raw[];
  const uint32_t raw = smem_u32(bs_raw);
  uint8_t* sm = bs_raw + (((raw + 1023u) & ~1023u) - raw);
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + 12 * A2_SLOT);
  uint64_t* ebar = bar + 12;
  const int tid = threadIdx.x, warp = tid >> 5;
  if (tid == 0) {
    for (int s = 0; s < nslot; ++s) { mbar_init(&bar[s], 1); mbar_init(&ebar[s], 8); }
    fence_mbar_init();
    prefetch_tmap(&map);
  }
  __syncthreads();
  // box coordinates advance without divisions: (row box, block) of the i-th box of this CTA
  int rb = static_cast<int>((static_cast<long long>(blockIdx.x) * nboxes) % row_boxes);
  int blk = static_cast<int>(((static_cast<long long>(blockIdx.x) * nboxes) / row_boxes) % blocks);
  auto issue = [&](int s) {
    mbar_expect_tx(&bar[s], A2_SLOT);
    tma_load_3d(sm + s * A2_SLOT, &map, &bar[s], 0, rb * 128, blk);
    if (++rb == row_boxes) { rb = 0; if (++blk == blocks) blk = 0; }
  };
  unsigned int acc = 0;
  if (mode & 2) {
    if (warp == 8) {
      if ((tid & 31) == 0) {
        for (int i = 0; i < nboxes; ++i) {
          const int s = i % nslot;
          if (i >= nslot) mbar_wait(&ebar[s], static_cast<uint32_t>(((i / nslot) - 1) & 1));
          issue(s);
        }
      }
    } else {
      for (int i = 0; i < nboxes; ++i) {
        const int s = i % nslot;
        if ((tid & 31) == 0) mbar_wait(&bar[s], static_cast<uint32_t>((i / nslot) & 1));
        __syncwarp();
        acc += *reinterpret_cast<const unsigned int*>(sm + s * A2_SLOT + tid * 64);
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(&ebar[s]);
      }
    }
  } else {
    // every thread keeps the coordinate counters in step; thread 0 / the rotating thread issues
    if (tid == 0) for (int i = 0; i < nslot && i < nboxes; ++i) issue(i);
    else for (int i = 0; i < nslot && i < nboxes; ++i) { if (++rb == row_boxes) { rb = 0; if (++blk == blocks) blk = 0; } }
    for (int i = 0; i < nboxes; ++i) {
      const int s = i % nslot;
      const uint32_t par = static_cast<uint32_t>((i / nslot) & 1);
      if (warp < 8) {
        if (mode & 1) { mbar_wait(&bar[s], par); }
        else { if ((tid & 31) == 0) mbar_wait(&bar[s], par); __syncwarp(); }
        acc += *reinterpret_cast<const unsigned int*>(sm + s * A2_SLOT + tid * 64);
      }
      __syncthreads();
      if (i + nslot < nboxes) {
        if (tid == (((i + nslot) & 7) << 5)) issue(s);
        else if (++rb == row_boxes) { rb = 0; if (++blk == blocks) blk = 0; }
      }
    }
  }
  if (acc == 0x12345678u) sink[0] = acc;
}

}  // namespace pq

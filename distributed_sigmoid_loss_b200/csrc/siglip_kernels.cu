// sm_90a kernels of the distributed sigmoid (SigLIP) loss hot path.
//
// What the reference does per text chunk (distributed_sigmoid_loss.py:22-33, rwightman_sigmoid_loss.py:49-66):
//     logits = img @ txt_chunk.T * exp(t') + b ; loss = -logsigmoid(labels * logits).sum()
// and, through autograd, two more contractions (G @ txt, G.T @ img) for the gradients.
//
// Here every contraction is a tile loop on the Hopper tensor cores (wgmma), one persistent warp-specialised kernel:
//   * 12 warps: two consumer warpgroups (each owns 64 rows of the 128 x 128 fp32 accumulator tile in registers: it
//     issues the wgmma's of its half and then runs the epilogue on those registers), a TMA producer warp, an idle
//     warp that initialises the barriers, and 2 auxiliary warps (NVSwitch peer pulls / folds, operand conversion);
//   * operands staged by TMA into a 128B-swizzled shared-memory ring guarded by full / empty mbarriers;
//   * kModeLoss: the epilogue turns the S tile into softplus / sigma terms, reduces the three scalar sums and
//     (training) writes the sigma tile as the scaled-fp16 operand of the gradient contractions through TMA stores —
//     the logits never exist in HBM;
//   * kModeOut: the epilogue scales the accumulator by grad_out * exp(t') / B, adds the fp32 positive-pair rank-1
//     term and writes fp32 or bf16 gradients. Two problems (dimg and dtxt) share one launch so that the tile count
//     fills the 132 SMs evenly.
// Instantiated for clusters of 1, 2 or 4 CTAs on vertically adjacent 128-row blocks: the CTAs of a cluster compute the
// same column tile, each fetches 1 / cluster of the common B tile and TMA-multicasts it to all of them.
#include "siglip_kernels.cuh"

#include <stdio.h>
#include <stdlib.h>

namespace siglip {

namespace {

constexpr int kBlockM = 128;   // accumulator rows per CTA (two consumer warpgroups x 64)
constexpr int kTileN = 128;    // accumulator columns per tile (= wgmma N)
constexpr int kBlockK = 64;    // 64 16-bit values = one 128-byte swizzle row
constexpr int kMmaK = 16;
constexpr int kNumEpiWarps = 8;                        // the two consumer warpgroups
constexpr int kProducerWarp = kNumEpiWarps;
constexpr int kInitWarp = kNumEpiWarps + 1;
constexpr int kAuxWarp = kNumEpiWarps + 2;             // this warp and the next run the auxiliary jobs
constexpr int kNumThreads = (kNumEpiWarps + 4) * 32;

constexpr int kStagingBytesPerWarp = 1024;  // one 16x32 16-bit slab, 64-byte rows, 64B-swizzled (TMA store source)

// Gradient kernel with 256-column tiles (wgmma m64n256, 128 accumulator registers per consumer thread): 48 KiB per
// stage, so 4 stages. The consumers fit the even split of __launch_bounds__(384, 1), 168 registers per thread.
constexpr int kWideTileN = kWideTileCols;
constexpr int kWideStages = 4;

// the loss-kernel modes that contract the teacher's operands (tmA1 / tmB1) before the student's
__host__ __device__ constexpr bool teacher_mode(int mode) { return mode == kModeDistill || mode == kModeDistillOpts; }

template <int kMode, int kStagesT, int kTileNT = kTileN>
struct Cfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;            // 16 KiB
  static constexpr int kBBytes = kTileNT * kBlockK * 2;            // 16 KiB (32 KiB for 256-column tiles)
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = kStagesT;
  static constexpr int kStagingBytes = (kMode != kModeOut) ? kNumEpiWarps * kStagingBytesPerWarp : 0;
  // kModeDistill, kModeDistillOpts: the teacher's probabilities (fp32, one 128 x 128 tile) follow the barrier block
  static constexpr int kPBytes = teacher_mode(kMode) ? kBlockM * kTileNT * 4 : 0;
  static constexpr int kSmemBytes =
      kStages * kStageBytes + kStagingBytes + 1024 /*barriers, reduction*/ + kPBytes + 1024 /*alignment slack*/;
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
};

constexpr float kLog2e = 1.4426950408889634f;

// log1p(e) / e on [0, 1], degree-7 interpolant at Chebyshev nodes; max relative error 3.2e-7 in fp32 Horner form.
// (lg2.approx has 2^-22 ABSOLUTE error near 1, i.e. ~4e-3 relative on log1p(4.5e-5) — not usable here.)
__device__ __forceinline__ float log1p_over_e(float e) {
  float p = -0.00837115291506052f;
  p = fmaf(p, e, 0.04349390044808388f);
  p = fmaf(p, e, -0.1068500280380249f);
  p = fmaf(p, e, 0.1768747717142105f);
  p = fmaf(p, e, -0.24474774301052094f);
  p = fmaf(p, e, 0.3327192962169647f);
  p = fmaf(p, e, -0.49997174739837646f);
  p = fmaf(p, e, 0.9999997615814209f);
  return p;
}

// two fp32 -> one 32-bit word of two 16-bit floats (low half = lo). kF16: IEEE fp16, else bf16.
template <bool kF16>
__device__ __forceinline__ uint32_t pack_16x2(float lo, float hi) {
  uint32_t r;
  if constexpr (kF16) {
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  } else {
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  }
  return r;
}

// fp16(lo * scale), fp16(hi * scale) in one word (low half = lo), scale > 0: the operand conversions. A finite value
// saturates at +-65504 (.satfinite: what clamping to the fp16 range before cvt.rn gave, product overflow included), NaN
// stays NaN, and +-inf stays +-inf, so a non-finite embedding entry reaches the loss and the gradients. .satfinite maps
// +-inf to +-65504 (0x7bff / 0xfbff), one below the infinities' bits (0x7c00 / 0xfc00): an infinite input adds that one.
// A clamp with fminf / fmaxf would return the non-NaN operand and turn NaN into -65504.
__device__ __forceinline__ uint32_t pack_f16x2_scaled(float lo, float hi, float scale) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi * scale), "f"(lo * scale));
  const uint32_t inf_lo = (__float_as_uint(lo) & 0x7fffffffu) == 0x7f800000u;
  const uint32_t inf_hi = (__float_as_uint(hi) & 0x7fffffffu) == 0x7f800000u;
  return r + inf_lo + (inf_hi << 16);
}

__device__ __forceinline__ void named_barrier_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// sum += x with a running compensation term (Kahan): the error of each fp32 addition is carried into the next one.
// Written with explicit intrinsics so that fast-math style reassociation cannot remove the compensation.
__device__ __forceinline__ void kahan_add(float& sum, float& comp, float x) {
  const float y = __fsub_rn(x, comp);
  const float t = __fadd_rn(sum, y);
  comp = __fsub_rn(__fsub_rn(t, sum), y);
  sum = t;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Bounded wait of the two auxiliary warps (64 threads) of a CTA on `n` consecutive flags written by peer GPUs
// (st.release.sys): ONE thread per CTA polls (acquire, system scope) with a back-off — thousands of threads hammering
// one L2 line slowed the MMA operand traffic of the whole kernel — then the 64 threads meet on a named barrier.
// Traps after timeout_ns (SIGLIP_OPT_PEER_TIMEOUT_MS: minutes by default, like a process-group timeout — a peer may
// legitimately be late by a checkpoint save or an evaluation pass).
__device__ __forceinline__ void wait_peer_flags(const volatile unsigned int* flags, int n, unsigned int value,
                                                unsigned long long timeout_ns, DebugRecord* dbg, unsigned int site) {
  if (threadIdx.x == kAuxWarp * 32) {
    uint64_t t0 = 0;
    uint32_t spins = 0;
    for (int f = 0; f < n; ++f) {
      while (true) {
        unsigned int v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + f) : "memory");
        if (v >= value) break;
        __nanosleep(200);
        if ((++spins & 0xffu) == 0) {
          const uint64_t now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          if (now - t0 > timeout_ns) {
            if (dbg != nullptr) {
              dbg->block = blockIdx.x;
              dbg->thread = static_cast<unsigned int>(f);
              dbg->aux0 = v;
              dbg->aux1 = value;
              dbg->code = site;
              __threadfence_system();
            }
            __trap();
          }
        }
      }
    }
    __threadfence();  // order the peer data reads of the other 63 threads after the observed flags
  }
  asm volatile("bar.sync 2, 64;" ::: "memory");
}

// Every CTA has finished its share of something: the last one to arrive (ticket) publishes. Called by ONE thread per
// CTA after a barrier that covers the CTA's writers; returns true on the last CTA. The ticket is left at zero.
__device__ __forceinline__ bool last_cta_arrives(unsigned int* ticket) {
  __threadfence_system();                     // this CTA's writes (possibly read by peers over NVLink) before the ticket
  const unsigned int t = atomicAdd(ticket, 1u);
  if (t != gridDim.x - 1) return false;
  atomicExch(ticket, 0u);                     // ready for the next launch
  __threadfence_system();                     // the other CTAs' writes (observed through the ticket) before the signal
  return true;
}

__device__ __forceinline__ void release_store_sys(unsigned int* flag, unsigned int value) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
}

// 16-byte load of peer (NVLink-mapped) or streaming data: no L1 allocation, data is touched once
__device__ __forceinline__ uint4 ld_peer_16(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// t' as the module holds it: fp64 like the reference's parameter (distributed_sigmoid_loss.py:11), or fp32
__device__ __forceinline__ float load_t_prime(const KernelParams& p) {
  return p.tprime_f64 ? static_cast<float>(*reinterpret_cast<const double*>(p.t_prime)) : *p.t_prime;
}

struct TileCoord {
  int prob;
  int m_blk;
  int n_blk;
  int part;    // -1: whole tile; 0 .. sk_parts-1: this work item is one K-slice of a split tile (0 = the owner, which
               // adds the other slices' partial accumulators and runs the epilogue)
  int slot;    // split tiles only: index into the partial-accumulator workspace / arrival counters
};

// Work unit of a cluster: kCS vertically adjacent 128-row blocks (same n block, consecutive m blocks) — one per CTA of
// the cluster, so that the B operand tile is common and can be TMA-multicast. tiles_m counts such row panels.
__device__ __forceinline__ int cluster_tiles(const Problem& pr) { return pr.tiles_m * pr.tiles_n; }

// Work item -> tile. Items 0 .. sk_first-1 are whole tiles in schedule order; with split-K (out kernel) the remaining
// sk_tiles tiles — the ragged last wave — appear sk_parts times, slice-major, so that the slices of one tile run on
// different clusters at the same time.
template <int kCS>
__device__ __forceinline__ TileCoord decode_tile(const KernelParams& p, int t, int crank) {
  TileCoord c;
  c.part = -1;
  c.slot = 0;
  if (p.sk_parts > 1 && t >= p.sk_first) {
    const int q = t - p.sk_first;
    c.part = q / p.sk_tiles;
    c.slot = q - c.part * p.sk_tiles;
    t = p.sk_first + c.slot;
  }
  const int t0 = cluster_tiles(p.prob[0]);
  c.prob = (t >= t0) ? 1 : 0;
  const int tt = c.prob ? t - t0 : t;
  const int tn = p.prob[c.prob].tiles_n;
  const int mrow = tt / tn;
  c.m_blk = mrow * kCS + crank;   // may lie beyond M in the last row panel: fully masked block
  c.n_blk = tt - mrow * tn;
  return c;
}

// k-blocks [kb0, kb1) of a work item: everything, or the item's slice of a split tile
__device__ __forceinline__ void item_k_range(const KernelParams& p, const TileCoord& tc, int num_kb, int& kb0,
                                             int& kb1) {
  if (tc.part < 0) {
    kb0 = 0;
    kb1 = num_kb;
  } else {
    kb0 = static_cast<int>(static_cast<long long>(num_kb) * tc.part / p.sk_parts);
    kb1 = static_cast<int>(static_cast<long long>(num_kb) * (tc.part + 1) / p.sk_parts);
  }
}

// -------------------------------------------------------------------------------------------------
// Accumulator fragment of a consumer thread (wgmma m64n128 f32): acc[4 i + e] holds row r_lo + 8 (e >> 1) and column
// 8 i + c_lo + (e & 1) of its warpgroup's 64 x 128 block, with r_lo = 16 (warp % 4) + lane / 4, c_lo = 2 (lane % 4).
// The epilogues walk it in slabs of 32 columns (acc[16 c .. 16 c + 15]): per warp a 16-row x 32-column block.
//
// Epilogue of the loss kernel. Per element (s = <img_i, txt_j>, z = t*s + b, reference distributed_sigmoid_loss.py:24-33):
//   negative pair: term = softplus(z),  g = dterm/dz = sigma(z)
//   positive pair: term = softplus(-z), g = -sigma(-z)            (own chunk diagonal only)
// Sums kept per thread: sum term, sum g, sum g*s (-> loss, dbias, dt').
//
// Fast path (whole warp slab has z < kFastZ, i.e. e = exp(z) < 2^-6, which is where a SigLIP batch lives:
// bias ~ -10): 1 MUFU (ex2) + ~8 FMA-pipe instructions per element, sigma and log1p by their series.
// General path: any z, exp(-|z|) + degree-7 log1p polynomial + rcp.
// -------------------------------------------------------------------------------------------------
constexpr float kFastZ = -4.2f;  // e < 0.015 < 2^-6: series truncated after e^2, relative error < e^3 = 3.4e-6

// The sigma slab goes to HBM through shared memory + one TMA store per warp: 8 conflict-free 4-byte st.shared per
// thread (64B swizzle) instead of 8 scattered 4-byte global stores.
struct GStore {
  const CUtensorMap* tmap;  // 16-bit [B, B] tensor, box {32 cols, 16 rows}, SWIZZLE_64B
  uint32_t stage;           // this warp's 1 KiB staging buffer (shared::cta address, 512-byte aligned)
  int row0;                 // first row of this warp's 16-row band
  int lane;
  uint64_t policy;          // L2 evict_first: the sigma lines are not read again before they have left the L2
};

// packed[2 j + h]: the two sigma values of column pair j (columns 8 j + c_lo, + 1) in row r_lo + 8 h of the band
__device__ __forceinline__ void store_g_slab(const GStore& gs, int col0, const uint32_t (&packed)[8]) {
  // the previous TMA store of this warp must have finished READING the staging buffer
  if (gs.lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  __syncwarp();
#pragma unroll
  for (uint32_t h = 0; h < 2; ++h) {
    const uint32_t r = (static_cast<uint32_t>(gs.lane) >> 2) + 8u * h;
    const uint32_t sw = (r >> 1) & 3u;   // 64B swizzle: 16-byte chunk ^= (row / 2) % 4
#pragma unroll
    for (uint32_t j = 0; j < 4; ++j) {
      const uint32_t addr = gs.stage + r * 64u + ((j ^ sw) << 4) + 4u * (static_cast<uint32_t>(gs.lane) & 3u);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(packed[2 * j + h]) : "memory");
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA engine
  __syncwarp();
  if (gs.lane == 0) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], %4;" ::"l"(
                     reinterpret_cast<uint64_t>(gs.tmap)),
                 "r"(gs.stage), "r"(col0), "r"(gs.row0), "l"(gs.policy)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}

// Weight of fragment element i = 4 j + 2 h + e1 (row half h, column 8 j + e1) of a slab (SIGLIP_OPT_SAMPLE_WEIGHTS):
// the thread's row weight times the column weight cw[2 j + e1]
__device__ __forceinline__ float slab_w(int i, const float* cw, float rw0, float rw1) {
  return (((i >> 1) & 1) ? rw1 : rw0) * cw[2 * (i >> 2) + (i & 1)];
}

// Fast path: every z of the slab is < kFastZ, so e = exp(z) < 2^-6 and both sigma(z) = e / (1 + e) and log1p(e) are
// evaluated by their alternating series on the FMA pipe (truncation < 3.4e-6 relative at the edge of the path, < 1e-8
// for the z ~ -10 of a SigLIP batch; the tolerance is 1e-3). One MUFU (ex2) per element instead of two: the epilogue
// is bound by the MUFU and FMA pipes.
// kW (SIGLIP_OPT_SAMPLE_WEIGHTS): element i has weight slab_w(i, cw, rw0, rw1); it scales e where e multiplies into both
// terms, so a weight of exactly 1 leaves every value bit-identical to the unweighted path.
// kL (per-sample losses, kModeSampleLoss): element i's term w softplus(z), computed next to the fmaf chain of the sum
// (which it leaves untouched), is added to lrow[row half] and lcol[2 j + e1] (the thread's 2 rows and 8 columns).
template <bool kW = false, bool kL = false>
__device__ __forceinline__ void loss_slab_fast(const float* v, float tl, float bl, int col0, bool store_g,
                                               const GStore& gst, float gscale, float& acc_sp, float& acc_g,
                                               float& acc_gs, const float* cw = nullptr, float rw0 = 1.f,
                                               float rw1 = 1.f, float* lrow = nullptr, float* lcol = nullptr) {
  uint32_t packed[8];
  float a_sp = 0.f, a_g = 0.f, a_gs = 0.f;
  float g_prev = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float s = v[i];
    const float e = ex2_approx(fmaf(s, tl, bl));        // exp(z), z < kFastZ
    float ew = e;
    if constexpr (kW) ew = e * slab_w(i, cw, rw0, rw1);
    // sigma is produced already multiplied by the power-of-two scale of the 16-bit operand (exact), and the two sums
    // that use it are un-scaled once per slab
    float q = fmaf(e, gscale, -gscale);                  // S sigma(z) / e = S (1 - e + e^2)  [- e^3 < 3.8e-6 dropped]
    q = fmaf(e, q, gscale);
    const float g = ew * q;                              // S sigma(z) (x w)
    float l = fmaf(e, 0.33333334f, -0.5f);               // log1p(e) / e = 1 - e/2 + e^2/3    [- e^3/4 < 1e-6 dropped]
    l = fmaf(e, l, 1.0f);
    a_sp = fmaf(ew, l, a_sp);
    if constexpr (kL) {
      const float term = ew * l;
      lrow[(i >> 1) & 1] += term;
      lcol[2 * (i >> 2) + (i & 1)] += term;
    }
    a_g += g;
    a_gs = fmaf(g, s, a_gs);
    // element i = 4 j + e': row half e' >> 1, column e' & 1 -> packed[2 j + (e' >> 1)]
    if (i & 1)
      packed[2 * (i >> 2) + ((i >> 1) & 1)] = pack_16x2<true>(g_prev, g);
    else
      g_prev = g;
  }
  const float inv_s = 1.0f / gscale;
  acc_sp += a_sp;
  acc_g = fmaf(a_g, inv_s, acc_g);
  acc_gs = fmaf(a_gs, inv_s, acc_gs);
  if (store_g) store_g_slab(gst, col0, packed);
}

// General path. row_lo: global row of this thread's first fragment row; col0: global column of the slab; c_lo as above.
// pos (kMask only): bit i set = element i is a positive pair by sample id (SIGLIP_OPT_SAMPLE_IDS); 0 without ids.
// kW: element i's weight multiplies its three terms once its label is applied (x * 1 == x: unit weights change no bit).
// kL: element i's term (sp once masked and weighted) is also added to lrow / lcol as in loss_slab_fast.
// kX (kModeGroups, with kMask): excl bit i set = element i is an excluded pair (same group, not a positive): its sp, g
// and stored sigma are 0, so it adds nothing anywhere. A positive is never excluded (the label tests come first).
template <bool kMask, bool kW = false, bool kL = false, bool kX = false>
__device__ __forceinline__ void loss_slab(const float* v, float t, float b, int row_lo, int col0, int c_lo, int nrows,
                                          int ncols, bool store_g, const GStore& gst, float gscale, float* g_diag,
                                          bool on_diag, uint32_t pos, float& acc_sp, float& acc_g, float& acc_gs,
                                          const float* cw = nullptr, float rw0 = 1.f, float rw1 = 1.f,
                                          float* lrow = nullptr, float* lcol = nullptr, uint32_t excl = 0u) {
  uint32_t packed[8];
  float g_prev = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int row = row_lo + 8 * ((i >> 1) & 1);
    const int col = col0 + 8 * (i >> 2) + c_lo + (i & 1);
    const float s = v[i];
    const float z = fmaf(s, t, b);
    const float e = ex2_approx(-fabsf(z) * kLog2e);    // exp(-|z|) in (0, 1]
    const float l = e * log1p_over_e(e);               // log1p(exp(-|z|))
    const float r = rcp_approx(1.0f + e);              // sigma(|z|)
    const float sig_z = (z >= 0.f) ? r : e * r;        // sigma(z)
    float sp = fmaxf(z, 0.f) + l;                      // softplus(z): negative pair (label -1)
    float g = sig_z;                                   // d softplus(z) / dz
    float g_store = sig_z;
    bool valid = true;
    if constexpr (kMask) {
      valid = (row < nrows) && (col < ncols);
      if (on_diag && row == col) {                     // positive pair (label +1): softplus(-z), -sigma(-z)
        sp = fmaxf(-z, 0.f) + l;
        g = -((z >= 0.f) ? e * r : r);                 // sigma(-z) without the 1 - sigma(z) cancellation
        g_store = 0.f;                                 // the own diagonal stays out of the 16-bit operand
        if (store_g && valid) {
          if constexpr (kW)
            g_diag[row] = g * slab_w(i, cw, rw0, rw1);
          else
            g_diag[row] = g;
        }
      } else if ((pos >> i) & 1u) {                    // any other positive (same sample id): same terms, and its
        sp = fmaxf(-z, 0.f) + l;                       // g * 2^14 in [-16384, 0) goes into the fp16 operand
        g = -((z >= 0.f) ? e * r : r);
        g_store = g;
      } else if (kX && ((excl >> i) & 1u)) {           // excluded pair (same group): neither pulled nor pushed
        sp = 0.f;
        g = 0.f;
        g_store = 0.f;
      }
      sp = valid ? sp : 0.f;
      g = valid ? g : 0.f;
      g_store = valid ? g_store : 0.f;
    }
    if constexpr (kW) {
      const float w = slab_w(i, cw, rw0, rw1);
      sp *= w;
      g *= w;
      g_store *= w;
    }
    acc_sp += sp;
    if constexpr (kL) {
      lrow[(i >> 1) & 1] += sp;
      lcol[2 * (i >> 2) + (i & 1)] += sp;
    }
    acc_g += g;
    acc_gs = fmaf(g, s, acc_gs);
    if (i & 1)
      packed[2 * (i >> 2) + ((i >> 1) & 1)] = pack_16x2<true>(g_prev, g_store * gscale);
    else
      g_prev = g_store * gscale;
  }
  if (store_g) store_g_slab(gst, col0, packed);
}

// -------------------------------------------------------------------------------------------------
// Focal pair loss (kModeFocal). With m = z for a negative and m = -z for a positive (the logit of the wrong answer):
//   term = a_t sigma(m)^gamma softplus(m),   dterm/dm = a_t sigma(m)^gamma (gamma sigma(-m) softplus(m) + sigma(m)),
//   g = dterm/dz = dterm/dm for a negative, -dterm/dm for a positive,
// with sigma(m)^gamma = exp(-gamma softplus(-m)) from the softplus the term computes anyway: one more ex2 per element.
// The general path forms neither sigma(m) nor 1 - sigma(m) by a subtraction; the series path's 1 - sigma(z), with
// sigma(z) < 2^-6, does not cancel. gamma = 0 gives the SigLIP terms. Every element
// takes its weight (1 without weights) and adds its term to lrow / lcol, as loss_slab with kW and kL.
// -------------------------------------------------------------------------------------------------
// Series path: every element of the slab is a negative with z < kFastZ (the vote of loss_slab_fast), so e = exp(z) <
// 2^-6, sigma(z) and softplus(z) = log1p(e) take the series of loss_slab_fast, and sigma(z)^gamma = exp(gamma (z -
// log1p(e))) reuses the exponent of e: one more ex2 than loss_slab_fast.
__device__ __forceinline__ void focal_slab_fast(const float* v, float tl, float bl, float gamma, float a_neg, int col0,
                                                bool store_g, const GStore& gst, float gscale, float& acc_sp,
                                                float& acc_g, float& acc_gs, const float* cw, float rw0, float rw1,
                                                float* lrow, float* lcol) {
  uint32_t packed[8];
  float g_prev = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float s = v[i];
    const float x = fmaf(s, tl, bl);                     // z log2(e)
    const float e = ex2_approx(x);                       // exp(z), z < kFastZ
    const float sig = e * fmaf(e, e - 1.0f, 1.0f);       // sigma(z) = e (1 - e + e^2)
    const float l = e * fmaf(e, fmaf(e, 0.33333334f, -0.5f), 1.0f);   // softplus(z) = e (1 - e/2 + e^2/3)
    const float pw = ex2_approx(gamma * fmaf(-l, kLog2e, x));         // sigma(z)^gamma
    const float aw = a_neg * slab_w(i, cw, rw0, rw1) * pw;
    const float term = aw * l;
    const float g = aw * fmaf(gamma * (1.0f - sig), l, sig);
    acc_sp += term;
    lrow[(i >> 1) & 1] += term;
    lcol[2 * (i >> 2) + (i & 1)] += term;
    acc_g += g;
    acc_gs = fmaf(g, s, acc_gs);
    if (i & 1)
      packed[2 * (i >> 2) + ((i >> 1) & 1)] = pack_16x2<true>(g_prev, g * gscale);
    else
      g_prev = g * gscale;
  }
  if (store_g) store_g_slab(gst, col0, packed);
}

// General path: any z, the labels, masks and exclusions of loss_slab<true, true, true, true> (pos, excl, the own
// diagonal into g_diag, rows / columns past the problem masked to 0).
__device__ __forceinline__ void focal_slab(const float* v, float t, float b, float gamma, float a_pos, float a_neg,
                                           int row_lo, int col0, int c_lo, int nrows, int ncols, bool store_g,
                                           const GStore& gst, float gscale, float* g_diag, bool on_diag, uint32_t pos,
                                           uint32_t excl, float& acc_sp, float& acc_g, float& acc_gs, const float* cw,
                                           float rw0, float rw1, float* lrow, float* lcol) {
  uint32_t packed[8];
  float g_prev = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int row = row_lo + 8 * ((i >> 1) & 1);
    const int col = col0 + 8 * (i >> 2) + c_lo + (i & 1);
    const float s = v[i];
    const float z = fmaf(s, t, b);
    const float e = ex2_approx(-fabsf(z) * kLog2e);    // exp(-|z|) in (0, 1]
    const float l = e * log1p_over_e(e);               // log1p(exp(-|z|))
    const float r = rcp_approx(1.0f + e);              // sigma(|z|)
    const bool dg = on_diag && row == col;             // the own diagonal: its term goes to g_diag
    const bool y = dg || ((pos >> i) & 1u);
    const float m = y ? -z : z;
    const float pm = (m >= 0.f) ? r : e * r;           // sigma(m)
    const float qm = (m >= 0.f) ? e * r : r;           // sigma(-m) = 1 - sigma(m)
    const float spm = fmaxf(m, 0.f) + l;               // softplus(m)
    const float pw = ex2_approx(-gamma * kLog2e * (fmaxf(-m, 0.f) + l));   // sigma(m)^gamma = exp(-gamma softplus(-m))
    const bool valid = (row < nrows) && (col < ncols) && (y || !((excl >> i) & 1u));   // a positive is never excluded
    const float aw = valid ? (y ? a_pos : a_neg) * slab_w(i, cw, rw0, rw1) * pw : 0.f;
    const float sp = valid ? aw * spm : 0.f;
    const float gm = valid ? aw * fmaf(gamma * qm, spm, pm) : 0.f;
    const float g = y ? -gm : gm;
    if (dg && store_g && valid) g_diag[row] = g;
    const float g_store = dg ? 0.f : g;                // the own diagonal stays out of the 16-bit operand
    acc_sp += sp;
    lrow[(i >> 1) & 1] += sp;
    lcol[2 * (i >> 2) + (i & 1)] += sp;
    acc_g += g;
    acc_gs = fmaf(g, s, acc_gs);
    if (i & 1)
      packed[2 * (i >> 2) + ((i >> 1) & 1)] = pack_16x2<true>(g_prev, g_store * gscale);
    else
      g_prev = g_store * gscale;
  }
  if (store_g) store_g_slab(gst, col0, packed);
}

// -------------------------------------------------------------------------------------------------
// Distillation (kModeDistill). Per element, with p the teacher's probability of the pair and y its hard label:
//   q = (1 - lambda) y + lambda p,   term = softplus(z) - q z,   g = sigma(z) - q      (times the pair's weight)
// sigma and softplus take the series of loss_slab_fast in a 16x32 slab whose z are all < kFastZ (warp vote, as in the
// plain loss kernel) and the exact form in every other slab. The teacher's accumulator goes through the same functions
// (distill_slab_series, distill_sigma) on the same slab geometry, so a teacher equal to the student gives
// p == sigma(z) bit for bit, and g == 0 at lambda = 1.
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool distill_slab_series(const float* v, float t, float b) {
  float smax = v[0];
#pragma unroll
  for (int j = 1; j < 16; ++j) smax = fmaxf(smax, v[j]);
  return __all_sync(0xffffffffu, fmaf(smax, t, b) < kFastZ);   // z is monotone in s (t > 0)
}

__device__ __forceinline__ void distill_terms(float s, float t, float b, float tl, float bl, bool series, float& z,
                                              float& sig, float& l) {
  z = fmaf(s, t, b);
  if (series) {
    const float e = ex2_approx(fmaf(s, tl, bl));        // exp(z) < 2^-6
    sig = e * fmaf(e, e - 1.0f, 1.0f);                  // e (1 - e + e^2)
    l = e * fmaf(e, fmaf(e, 0.33333334f, -0.5f), 1.0f); // log1p(e) = e (1 - e/2 + e^2/3)
  } else {
    const float e = ex2_approx(-fabsf(z) * kLog2e);    // exp(-|z|)
    const float r = rcp_approx(1.0f + e);
    sig = (z >= 0.f) ? r : e * r;
    l = e * log1p_over_e(e);                           // softplus(z) - max(z, 0)
  }
}

__device__ __forceinline__ float distill_sigma(float s, float t, float b, float tl, float bl, bool series) {
  float z, sig, l;
  distill_terms(s, t, b, tl, bl, series, z, sig, l);
  return sig;
}

// Thread-private fp32 slot of fragment element i in the teacher-probability buffer: element-major, so that the 256
// consumer threads touch 256 consecutive words (no bank conflicts) and each reads back only what it wrote.
__device__ __forceinline__ uint32_t distill_p_addr(uint32_t pbuf, int i) {
  return pbuf + 4u * (static_cast<uint32_t>(i) * (kNumEpiWarps * 32u) + threadIdx.x);
}

// One 16x32 slab of the distillation epilogue. kMask: rows / columns past the matrix are dropped and labels are applied
// (the own-chunk diagonal, whose g goes to g_diag in fp32, and the pos bits of sample ids or label sets); without it
// y = 0. w: per-sample weights (cw / rw0 / rw1 as in slab_w) when non-zero.
// kL (kModeDistillOpts): element i's term, once weighted and masked, is also added to lrow / lcol as in loss_slab.
// kX (kModeDistillOpts, with kMask): excl bit i set = element i is an excluded pair (same group, not a positive): it is
// masked like a pair past the matrix, so its term, g and stored sigma are 0 whatever its teacher probability.
template <bool kMask, bool kL = false, bool kX = false>
__device__ __forceinline__ void distill_slab(const float* v, uint32_t pbuf, int c, float t, float b, float tl, float bl,
                                             float lambda, int row_lo, int col0, int c_lo, int nrows, int ncols,
                                             bool store_g, const GStore& gst, float gscale, float* g_diag, bool on_diag,
                                             uint32_t pos, bool w, const float* cw, float rw0, float rw1,
                                             float& acc_sp, float& acc_g, float& acc_gs, float* lrow = nullptr,
                                             float* lcol = nullptr, uint32_t excl = 0u) {
  uint32_t packed[8];
  float g_prev = 0.f;
  const float one_minus = 1.0f - lambda;
  const bool series = distill_slab_series(v, t, b);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float s = v[i];
    float pt;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(pt) : "r"(distill_p_addr(pbuf, 16 * c + i)));
    float z, sig, l;
    distill_terms(s, t, b, tl, bl, series, z, sig, l);
    float y = 0.f;
    bool valid = true, own_diag = false;
    int row = 0;
    if constexpr (kMask) {
      row = row_lo + 8 * ((i >> 1) & 1);
      const int col = col0 + 8 * (i >> 2) + c_lo + (i & 1);
      valid = (row < nrows) && (col < ncols);
      own_diag = on_diag && row == col;
      y = (own_diag || ((pos >> i) & 1u)) ? 1.0f : 0.f;
      if constexpr (kX) valid = valid && (own_diag || !((excl >> i) & 1u));   // excl never holds a pos bit
    }
    const float q = fmaf(lambda, pt, one_minus * y);
    float sp = ((z >= 0.f) ? (1.0f - q) * z : -q * z) + l;   // softplus(z) - q z without cancelling at q = 1
    float g = sig - q;
    if (w) {
      const float wi = slab_w(i, cw, rw0, rw1);
      sp *= wi;
      g *= wi;
    }
    float g_store = g;
    if constexpr (kMask) {
      if (own_diag) {                                  // the own diagonal stays out of the 16-bit operand
        if (store_g && valid) g_diag[row] = g;
        g_store = 0.f;
      }
      sp = valid ? sp : 0.f;
      g = valid ? g : 0.f;
      g_store = valid ? g_store : 0.f;
    }
    acc_sp += sp;
    if constexpr (kL) {
      lrow[(i >> 1) & 1] += sp;
      lcol[2 * (i >> 2) + (i & 1)] += sp;
    }
    acc_g += g;
    acc_gs = fmaf(g, s, acc_gs);
    if (i & 1)
      packed[2 * (i >> 2) + ((i >> 1) & 1)] = pack_16x2<true>(g_prev, g_store * gscale);
    else
      g_prev = g_store * gscale;
  }
  if (store_g) store_g_slab(gst, col0, packed);
}

// -------------------------------------------------------------------------------------------------
// In-batch retrieval metrics (kMetrics): the argmax of every row and column of the logits, from the accumulator tile.
// Key of a candidate: (order-preserving bits of s) << 32 | (0xFFFFFFFF - global index). The unsigned max of two keys is
// the larger s, ties to the lower index; 0 is "no candidate" (every real key is larger). z = t s + b is monotone in s
// (t > 0), so the ranking of z is the ranking of s. The accumulator is s itself, or s * 2^8 for the fp16 x 16
// operands: a power-of-two scale changes neither the order nor the ties.
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long metric_key(float s, int gidx) {
  const uint32_t u = __float_as_uint(__fadd_rn(s, 0.0f));     // -0 -> +0: equal values must tie on the index
  const uint32_t ord = u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u);
  return (static_cast<unsigned long long>(ord) << 32) | (0xFFFFFFFFu - static_cast<uint32_t>(gidx));
}

__device__ __forceinline__ unsigned long long max_u64(unsigned long long a, unsigned long long b) { return a > b ? a : b; }

__device__ __forceinline__ void red_max_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Row side: per fragment row, the best of the thread's 32 columns (strict > in increasing column order keeps the lowest
// index), then the quad that holds the row (shfl_xor 1, 2), then one red.max per row and tile.
// Column side, per 32-column slab: the better of the thread's 2 rows for each of its 8 columns, then a reduce-scatter over
// the warp's 8 row groups (lanes xor 16, 8, 4) that leaves lane l with column q = l >> 2 of the 8 its lane % 4 group
// holds, then one red.max per lane and slab. Rows >= M and columns >= N are never candidates.
__device__ __forceinline__ void tile_metrics(const float (&acc)[64], int row_lo, int col_base, int c_lo, int M, int N,
                                             int lane, const KernelParams& p) {
  float best0 = -INFINITY, best1 = -INFINITY;
  int bc0 = -1, bc1 = -1;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    if (i & 2) continue;   // element i (row r_lo) and i + 2 (row r_lo + 8) share the column
    const int col = col_base + 8 * (i >> 2) + c_lo + (i & 1);
    if (col < N) {
      if (acc[i] > best0) { best0 = acc[i]; bc0 = col; }
      if (acc[i + 2] > best1) { best1 = acc[i + 2]; bc1 = col; }
    }
  }
  unsigned long long k0 = (bc0 >= 0) ? metric_key(best0, p.col_off + bc0) : 0ull;
  unsigned long long k1 = (bc1 >= 0) ? metric_key(best1, p.col_off + bc1) : 0ull;
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    k0 = max_u64(k0, __shfl_xor_sync(0xffffffffu, k0, o));
    k1 = max_u64(k1, __shfl_xor_sync(0xffffffffu, k1, o));
  }
  if ((lane & 3) == 0) {
    if (row_lo < M && k0 != 0ull) red_max_u64(p.row_keys + row_lo, k0);
    if (row_lo + 8 < M && k1 != 0ull) red_max_u64(p.row_keys + row_lo + 8, k1);
  }
  const bool v0 = row_lo < M, v1 = row_lo + 8 < M;
#pragma unroll
  for (int c = 0; c < kTileN / 32; ++c) {
    // ck[q], q = 2 j + e: column 32 c + 8 j + c_lo + e of the tile
    unsigned long long ck[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int i = 16 * c + 4 * (q >> 1) + (q & 1);
      const float a = acc[i], b = acc[i + 2];
      const bool take_a = v0 && (!v1 || a >= b);   // tie: the lower row
      const int col = col_base + 32 * c + 8 * (q >> 1) + c_lo + (q & 1);
      ck[q] = (col < N && (v0 || v1)) ? metric_key(take_a ? a : b, p.row_off + (take_a ? row_lo : row_lo + 8)) : 0ull;
    }
    // reduce-scatter: after the step over lane bit m, ck[0 .. h) holds the columns q = k + (bit m of lane ? h : 0)
#pragma unroll
    for (int h = 4, m = 16; h >= 1; h >>= 1, m >>= 1) {
      const bool hi = (lane & m) != 0;
#pragma unroll
      for (int k = 0; k < h; ++k) {
        const unsigned long long send = hi ? ck[k] : ck[k + h];
        const unsigned long long keep = hi ? ck[k + h] : ck[k];
        ck[k] = max_u64(keep, __shfl_xor_sync(0xffffffffu, send, m));
      }
    }
    const int q = lane >> 2;   // bits 4, 3, 2 of the lane = 4, 2, 1 in q
    const int col = col_base + 32 * c + 8 * (q >> 1) + c_lo + (q & 1);
    if (col < N && ck[0] != 0ull) red_max_u64(p.col_keys + col, ck[0]);
  }
}

// -------------------------------------------------------------------------------------------------
// Top-K retrieval (kModeTopK): per row and per column a list of kTopKMax 64-bit keys (the metric keys above), sorted
// best first, of which the first K are filled; 0 = empty slot. A candidate c enters with a chain of atomic maxima:
// for s = 0 .. K-1, old = atom.max(&list[s], c), and if old < c the displaced key old is carried on instead; the chain
// ends when the carried key is 0. Every atomic keeps the larger key and carries the smaller, so no key is lost or
// duplicated, slots never decrease, and the list stays sorted; the keys are distinct, so whatever the order of the
// atomics the final list is exactly the top K of its candidates (DESIGN.md, "Top-K retrieval").
// Prefilter: a candidate not above the list's K-th slot cannot enter. That slot is read once per fragment row and tile
// and once per column and 32-column slab with a plain relaxed load (a stale value is a lower bound: slots only grow),
// and raised by what each chain learns (the key carried out of slot K-1 is below that slot).
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long atom_max_u64(unsigned long long* p, unsigned long long v) {
  unsigned long long old;
  asm volatile("atom.relaxed.gpu.global.max.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
  return old;
}

// volatile, so that it is read anew on every tile (consecutive tiles of a CTA share their rows: a pure load would be
// hoisted out of the tile loop); no memory clobber, so a slab's 8 loads issue back to back ahead of its chains
__device__ __forceinline__ unsigned long long topk_floor(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}

// Insert c into a list of k slots. Returns a key below the final list[k - 1], or 0 when the chain ended early.
__device__ __forceinline__ unsigned long long topk_insert(unsigned long long* list, int k, unsigned long long c) {
  for (int s = 0; s < k; ++s) {
    const unsigned long long old = atom_max_u64(list + s, c);
    if (old < c) {
      c = old;
      if (c == 0ull) return 0ull;
    }
  }
  return c;
}

// Rows: the concurrent clusters of a step work on the tiles of one row panel (the schedule is row-major), so a row's
// list has no useful floor yet when most of its tiles arrive. Each quad therefore selects its row's keys of the tile
// best first, one per round (round r: the quad's largest key below the one of round r - 1, shfl_xor 1, 2), and its
// first thread inserts it; the rounds stop at the list's floor, or after K. Columns, per 32-column slab: each thread
// offers its 2 rows of each of its 8 columns (a column's tiles arrive panel after panel, behind an established floor).
// Rows >= M and columns >= N are never candidates.
__device__ __forceinline__ void tile_topk(const float (&acc)[64], int row_lo, int col_base, int c_lo, int M, int N,
                                          int lane, const KernelParams& p) {
  const int k = p.tk_k;
  const bool v0 = row_lo < M, v1 = row_lo + 8 < M;
  const int lead = lane & ~3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool valid = h ? v1 : v0;
    const int row = min(row_lo + 8 * h, M - 1);
    unsigned long long thr = valid ? topk_floor(p.tk_rows + static_cast<size_t>(row) * kTopKMax + k - 1) : ~0ull;
    thr = __shfl_sync(0xffffffffu, thr, lead);   // one floor per quad
    // the previous round's key as (value, column): the scan compares the accumulator in place (64-bit keys of all 32
    // elements would be hoisted out of the rounds into registers); equal values order by column as the keys do
    // (+inf, -1): no bound in round 0; (-inf, INT_MAX): nothing selected. A NaN logit compares false and is never
    // selected here (the row side of a non-finite step is undefined)
    float bv = INFINITY;
    int bc = -1;
    for (int r = 0; r < k; ++r) {
      float cv = -INFINITY;
      int cc = 0x7fffffff;
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        if (((i >> 1) & 1) != h) continue;
        const int col = col_base + 8 * (i >> 2) + c_lo + (i & 1);
        const float v = acc[i];
        if (col < N && (v < bv || (v == bv && col > bc)) && (v > cv || (v == cv && col < cc))) {
          cv = v;
          cc = col;
        }
      }
      unsigned long long best = (cc != 0x7fffffff) ? metric_key(cv, p.col_off + cc) : 0ull;
      best = max_u64(best, __shfl_xor_sync(0xffffffffu, best, 1));
      best = max_u64(best, __shfl_xor_sync(0xffffffffu, best, 2));
      const bool go = best > thr;   // the same in the 4 threads of a quad
      if (!__any_sync(0xffffffffu, go)) break;
      if (go && lane == lead) thr = max_u64(thr, topk_insert(p.tk_rows + static_cast<size_t>(row) * kTopKMax, k, best));
      thr = __shfl_sync(0xffffffffu, thr, lead);
      if (go) {   // the next round looks below the key just taken
        const uint32_t ord = static_cast<uint32_t>(best >> 32);
        bv = __uint_as_float(ord ^ ((ord >> 31) ? 0x80000000u : 0xFFFFFFFFu));
        bc = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(best)) - p.col_off;
      } else {    // a quad that stopped offers nothing more
        bv = -INFINITY;
        bc = 0x7fffffff;
      }
    }
  }
#pragma unroll
  for (int c = 0; c < kTileN / 32; ++c) {
    unsigned long long thr[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int col = col_base + 32 * c + 8 * (q >> 1) + c_lo + (q & 1);
      thr[q] = (col < N) ? topk_floor(p.tk_cols + static_cast<size_t>(col) * kTopKMax + k - 1) : ~0ull;
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int col = col_base + 32 * c + 8 * (q >> 1) + c_lo + (q & 1);
      unsigned long long* list = p.tk_cols + static_cast<size_t>(min(col, N - 1)) * kTopKMax;
      const int i = 16 * c + 4 * (q >> 1) + (q & 1);
      if (v0) {
        const unsigned long long key = metric_key(acc[i], p.row_off + row_lo);
        if (key > thr[q]) thr[q] = max_u64(thr[q], topk_insert(list, k, key));
      }
      if (v1) {
        const unsigned long long key = metric_key(acc[i + 2], p.row_off + row_lo + 8);
        if (key > thr[q]) topk_insert(list, k, key);
      }
    }
  }
}

// Epilogue of the out kernel: one row of the fragment (h = 0: row_lo, 1: row_lo + 8), kN / 8 column pairs (16 for
// 128-column tiles, 32 for 256-column ones).
//   val = scale * (acc * acc_scale + fix * x[row, col]) (+ add_src[row, col]);  written as fp32 or bf16
// parts / nparts: owner of a split tile — the other K-slices' fp32 partials (float4 j of this thread's fragment at
// parts[j * 256], slices part_stride apart) are added to acc first, in slice order. (Read here instead of being added
// into the accumulator registers: a non-wgmma write to them makes ptxas serialise every wgmma of the kernel.)
// All global loads of a group of four column pairs are issued before its stores: the stores may alias the loads as far
// as the compiler knows, and a load -> store -> load chain exposes one L2 round trip per pair.
// fix_rows: rows of fix_mat; a row at or past it has no positive-pair term and reads nothing there (with hard negatives
// the dtxt problem's M = T exceeds the B rows of its fix_mat, the caller's image buffer).
template <int kN>
__device__ __forceinline__ void out_row(const float (&acc)[kN / 2], int h, float scale, int row, int col0, int c_lo,
                                       const Problem& pr, float fix, int fix_rows, const float4* parts = nullptr,
                                       int nparts = 0, size_t part_stride = 0) {
  if (row >= pr.M) return;
  const float as = pr.acc_scale;   // undoes the power-of-two scaling of the fp16 operands (1 for bf16)
  const float xs = (pr.fix_mat_scale != 0.f) ? pr.fix_mat_scale : 1.0f;
  const float fixs = fix * xs;
  const __nv_bfloat16* xrow =
      (pr.fix_mat != nullptr && row < fix_rows) ? pr.fix_mat + static_cast<long long>(row) * pr.ldx : nullptr;
  const float* arow = pr.add_src ? pr.add_src + static_cast<long long>(row) * pr.ld_add : nullptr;
#pragma unroll
  for (int jb = 0; jb < kN / 32; ++jb) {
    uint32_t xw[4];
    float2 ad[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int c = col0 + 8 * (4 * jb + jj) + c_lo;
      const bool in = c < pr.N;   // N % 8 == 0 (host): a column pair is wholly inside or outside
      xw[jj] = (xrow != nullptr && in) ? __ldg(reinterpret_cast<const unsigned int*>(xrow + c)) : 0u;
      ad[jj] = (arow != nullptr && in) ? *reinterpret_cast<const float2*>(arow + c) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = 4 * jb + jj;
      const int c = col0 + 8 * j + c_lo;
      if (c < pr.N) {
        float o0 = acc[4 * j + 2 * h], o1 = acc[4 * j + 2 * h + 1];
        for (int sp = 0; sp < nparts; ++sp) {     // fixed order: slice 0 (mine) + 1 + 2 + ...
          const float4 a = __ldcg(parts + static_cast<size_t>(sp) * part_stride + j * (kNumEpiWarps * 32));
          o0 += h ? a.z : a.x;
          o1 += h ? a.w : a.y;
        }
        o0 *= as;
        o1 *= as;
        if (xrow != nullptr) {
          float x0, x1;
          if (pr.fix_f16) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&xw[jj]));
            x0 = f.x;
            x1 = f.y;
          } else {
            x0 = __uint_as_float(xw[jj] << 16);
            x1 = __uint_as_float(xw[jj] & 0xffff0000u);
          }
          o0 = fmaf(fixs, x0, o0);
          o1 = fmaf(fixs, x1, o1);
        }
        o0 = fmaf(o0, scale, ad[jj].x);   // zeros without a running sum
        o1 = fmaf(o1, scale, ad[jj].y);
        if (pr.out_bf16) {
          __nv_bfloat16* orow = reinterpret_cast<__nv_bfloat16*>(pr.out) + static_cast<long long>(row) * pr.ldo;
          *reinterpret_cast<uint32_t*>(orow + c) = pack_16x2<false>(o0, o1);
        } else {
          float* orow = reinterpret_cast<float*>(pr.out) + static_cast<long long>(row) * pr.ldo;
          *reinterpret_cast<float2*>(orow + c) = make_float2(o0, o1);
        }
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------
// Mainloop of one consumer warpgroup: acc (+)= A[its 64 rows] * B[kN columns]^T over k-blocks [kb0, kb1), operands
// from the shared-memory ring. One k block = 4 wgmma's; the stage of the previous k block is handed back (to every CTA
// of the cluster that multicasts into it) once wgmma.wait_group says its MMAs have finished reading it.
// -------------------------------------------------------------------------------------------------
template <int kType, int kTA, int kTB, int kCS, int kStageBytes, int kN = kTileN>
__device__ __forceinline__ void mma_loop(float (&acc)[kN / 2], int kb0, int kb1, int& stage, uint32_t& phase, int nstages,
                                         uint64_t adesc0, uint64_t bdesc0, uint32_t a_adv, uint32_t b_adv,
                                         uint32_t full0, uint32_t empty0, int lane, DebugRecord* dbg, int t,
                                         long long* waited) {
  auto release = [&](int s) {
    if (lane == 0) {
      const uint32_t eb = empty0 + 8u * static_cast<uint32_t>(s);
      if constexpr (kCS == 1) {
        mbar_arrive(eb);
      } else {
#pragma unroll
        for (uint32_t r = 0; r < static_cast<uint32_t>(kCS); ++r) mbar_arrive_cluster_relaxed(mapa_shared(eb, r));
      }
    }
  };
#pragma unroll
  for (int i = 0; i < kN / 2; ++i) acc_fence(acc[i]);
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(full0 + 8u * static_cast<uint32_t>(stage), phase, dbg, 3, t, kb, 0, waited);
    const uint64_t so = static_cast<uint64_t>(stage) * static_cast<uint64_t>(kStageBytes >> 4);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / kMmaK; ++k) {
      if constexpr (kN == kWideTileN)
        wgmma_m64n256<kType, kTA, kTB>(acc, adesc0 + so + static_cast<uint64_t>(k * a_adv),
                                       bdesc0 + so + static_cast<uint64_t>(k * b_adv), (kb != kb0 || k != 0) ? 1u : 0u);
      else
        wgmma_m64n128<kType, kTA, kTB>(acc, adesc0 + so + static_cast<uint64_t>(k * a_adv),
                                       bdesc0 + so + static_cast<uint64_t>(k * b_adv), (kb != kb0 || k != 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<1>();   // the MMAs of the previous k block are done: its stage may be refilled
    if (prev >= 0) release(prev);
    prev = stage;
    if (++stage == nstages) {
      stage = 0;
      phase ^= 1u;
    }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < kN / 2; ++i) acc_fence(acc[i]);
  if (prev >= 0) release(prev);
}

// The same loop for e4m3 operands (K-major, 32 values per wgmma). Hopper's fp8 wgmma keeps its accumulator at reduced
// precision (~14 significant bits), so a chain of them drifts from the fp32 sum by ~1e-3 relative. Each instruction
// here starts from zero (scale-d = 0) and its result is added into the fp32 `sum` on the CUDA cores: the products of
// e4m3 values are exact, and only the sum of the 32 products of one instruction passes through the narrow accumulator.
// `acc` is only ever written by wgmma (a non-wgmma write to a wgmma accumulator makes ptxas serialise every wgmma of
// the kernel); `sum` is the result.
template <int kCS, int kStageBytes>
__device__ __forceinline__ void mma_loop_f8(float (&sum)[64], float (&acc)[64], int kb0, int kb1, int& stage,
                                            uint32_t& phase, int nstages, uint64_t adesc0, uint64_t bdesc0,
                                            uint32_t full0, uint32_t empty0, int lane, DebugRecord* dbg, int t,
                                            long long* waited) {
#pragma unroll
  for (int i = 0; i < 64; ++i) sum[i] = 0.f;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(full0 + 8u * static_cast<uint32_t>(stage), phase, dbg, 3, t, kb, 0, waited);
    const uint64_t so = static_cast<uint64_t>(stage) * static_cast<uint64_t>(kStageBytes >> 4);
#pragma unroll 1
    for (int k = 0; k < kBlockK / kMmaK; ++k) {   // 4 x 32 bytes of the 128-byte swizzle row
#pragma unroll
      for (int i = 0; i < 64; ++i) acc_fence(acc[i]);
      wgmma_fence();
      wgmma_m64n128<2, 0, 0>(acc, adesc0 + so + static_cast<uint64_t>(k * 2), bdesc0 + so + static_cast<uint64_t>(k * 2),
                             0u);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        acc_fence(acc[i]);
        sum[i] += acc[i];
      }
    }
    if (lane == 0) {   // this k block's MMAs are complete: hand the stage back
      const uint32_t eb = empty0 + 8u * static_cast<uint32_t>(stage);
      if constexpr (kCS == 1) {
        mbar_arrive(eb);
      } else {
#pragma unroll
        for (uint32_t r = 0; r < static_cast<uint32_t>(kCS); ++r) mbar_arrive_cluster_relaxed(mapa_shared(eb, r));
      }
    }
    if (++stage == nstages) {
      stage = 0;
      phase ^= 1u;
    }
  }
}

// Epilogue of the distillation loss kernel over one 128 x 128 tile: the loss kernel's slab walk (metric keys, masking,
// the own diagonal, sample ids and weights, now read at run time) with distill_slab in place of the hard-label slabs.
// The three sums go into the thread's compensated running sums.
__device__ __forceinline__ void distill_epilogue(const KernelParams& p, const float (&acc)[kTileN / 2], uint32_t pbuf,
                                                 const CUtensorMap* tmG, uint32_t staging_base, int warp, int wg,
                                                 int lane, int row0, int col_base, int row_lo, int c_lo,
                                                 const Problem& pr, float t_eff, float bias, float tl, float bl,
                                                 uint64_t policy, float& s_sp, float& c_sp, float& s_g, float& c_g,
                                                 float& s_gs, float& c_gs) {
  if (p.row_keys != nullptr) tile_metrics(acc, row_lo, col_base, c_lo, pr.M, pr.N, lane, p);
  float acc_sp = 0.f, acc_g = 0.f, acc_gs = 0.f;
  const bool edge = (row0 + kBlockM > pr.M) || (col_base + kTileN > pr.N);
  const bool diag = p.own_chunk && (row0 == col_base);
  const bool sg = p.store_g != 0;
  GStore gst;
  gst.tmap = tmG;
  gst.stage = staging_base + static_cast<uint32_t>(warp) * kStagingBytesPerWarp;
  gst.row0 = row0 + wg * 64 + (warp & 3) * 16;
  gst.lane = lane;
  gst.policy = policy;
  const bool ids = p.row_ids != nullptr, w = p.row_w != nullptr;
  int64_t rid0 = 0, rid1 = 0;
  uint32_t rpos = 0u;
  if (ids) {
    rid0 = p.row_ids[min(row_lo, pr.M - 1)];
    rid1 = p.row_ids[min(row_lo + 8, pr.M - 1)];
    rpos = (row_lo < p.row_pos_n ? 0x3333u : 0u) | (row_lo + 8 < p.row_pos_n ? 0xCCCCu : 0u);
  }
  float rw0 = 1.f, rw1 = 1.f;
  if (w) {
    rw0 = p.row_w[min(row_lo, pr.M - 1)];
    rw1 = p.row_w[min(row_lo + 8, pr.M - 1)];
  }
#pragma unroll
  for (int c = 0; c < kTileN / 32; ++c) {
    const float* v = acc + 16 * c;
    const int col0 = col_base + 32 * c;
    float cw[8];
    if (w) {
#pragma unroll
      for (int j = 0; j < 8; ++j) cw[j] = p.col_w[min(col0 + 8 * (j >> 1) + c_lo + (j & 1), pr.N - 1)];
    }
    const bool slab_diag = diag && (gst.row0 < col0 + 32) && (col0 < gst.row0 + 16);
    const bool slab_edge = edge && ((gst.row0 + 16 > pr.M) || (col0 + 32 > pr.N));
    uint32_t pos = 0;
    bool slab_pos = false;
    if (ids) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int e1 = 0; e1 < 2; ++e1) {
          const int col = col0 + 8 * j + c_lo + e1;
          if (col < p.col_pos_n) {
            const int64_t cid = p.col_ids[col];
            pos |= static_cast<uint32_t>(cid == rid0) << (4 * j + e1);
            pos |= static_cast<uint32_t>(cid == rid1) << (4 * j + 2 + e1);
          }
        }
      }
      pos &= rpos;
      slab_pos = __any_sync(0xffffffffu, pos != 0u);
    }
    // the series / exact choice is made per slab inside (distill_slab_series)
    if (!slab_edge && !slab_diag && !slab_pos)
      distill_slab<false>(v, pbuf, c, t_eff, bias, tl, bl, p.distill_lambda, row_lo, col0, c_lo, pr.M, pr.N, sg, gst,
                          p.g_scale, p.g_diag, false, 0u, w, cw, rw0, rw1, acc_sp, acc_g, acc_gs);
    else
      distill_slab<true>(v, pbuf, c, t_eff, bias, tl, bl, p.distill_lambda, row_lo, col0, c_lo, pr.M, pr.N, sg, gst,
                         p.g_scale, p.g_diag, slab_diag, pos, w, cw, rw0, rw1, acc_sp, acc_g, acc_gs);
  }
  kahan_add(s_sp, c_sp, acc_sp);
  kahan_add(s_g, c_g, acc_g);
  kahan_add(s_gs, c_gs, acc_gs);
}

// -------------------------------------------------------------------------------------------------
// Per-sample losses (kModeSampleLoss): row and column sums of the terms w_ij softplus(-y_ij z_ij) the loss adds up, from
// the same per-element values (loss_slab_fast / loss_slab with kL). Every partial is rounded once to a 64-bit
// fixed-point word (value * 2^32) and added with red.add.u64: integer addition is associative, so the sums depend only
// on the 128 x 128 tile and 16-row slab geometry, never on the order of the atomics, the cluster shape or the schedule.
// Every term is >= 0 (softplus, weights in [0, 1]). A partial that is not below kSampleLossMaxPartial (too large, +inf
// or NaN) is never added as a number: it ORs a poison bit into the word sl_poison words behind, which the finalisation
// decodes into +inf (1) or NaN (2).
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ void red_or_b64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.or.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// v * 2^32 is exact in fp32 and below 2^48, so the conversion to an integer does not round
__device__ __forceinline__ void sample_loss_add(unsigned long long* w, long long poison, float v) {
  if (v < kSampleLossMaxPartial) {   // false for NaN and +inf
    const unsigned long long q = __float2ull_rn(v * 4294967296.0f);
    if (q != 0ull) red_add_u64(w, q);
  } else {
    red_or_b64(w + poison, (v != v) ? 2ull : 1ull);
  }
}

// The loss epilogue of kModeSampleLoss. The three sums, g_diag and the stored sigma operand are those of the kModeLoss
// epilogue bit for bit: the same slab functions and path choices, with unit weights when the step has none (x * 1 == x)
// and the ids and metric keys as runtime options. On top:
//   rows:    each thread sums its two fragment rows over the tile's 4 slabs, the quad adds its 4 threads (shfl_xor 1, 2),
//            one red.add per row and tile;
//   columns: per slab, the thread's 2 rows of each of its 8 columns, then a reduce-scatter over the warp's 8 row groups
//            (lanes xor 16, 8, 4, as in tile_metrics) that leaves lane l with column q = l >> 2 of its lane % 4 group,
//            one red.add per lane and slab.
// Rows >= M and columns >= N add nothing (their terms are masked to 0 and their words do not exist).
// kTopK (kModeTopK): the top-K insertion (tile_topk) runs first, after the argmax keys, and the fixed-point sums are a
// runtime option (p.sl_rows); the three sums, g_diag and the sigma operand are unchanged.
// kGroups (kModeGroups): excluded same-group pairs (p.row_grp / p.col_grp). Once per tile the groups of the thread's two
// fragment rows, once per slab those of its 8 columns (clamped like the ids); the excl bits of the matching elements
// that are not positives, and a warp vote: a slab with an excluded element takes the masked path, which zeroes it, and
// every other slab keeps the path it takes without groups. Top-K lists and the per-sample sums are runtime options.
// kLabels (kModeLabels): positives from label sets (p.row_lab / p.col_lab, p.lab_m labels each). Once per tile, before
// the slab loop, each of the thread's two fragment rows' set is compared with the sets of its 32 columns (lab_m^2 64-bit
// compares per element; rolled loops, so that no set stays in registers across the loop), together with the id
// positives of the own chunk (own_pos_ids); the 64 pos bits are the only state the slab loop carries. There they form
// pos before the warp vote: a slab with a positive takes the masked path, every other slab keeps its path. Groups
// (tested after these positives), top-K lists and the per-sample sums are runtime options.
// kFocal (kModeFocal): the focal terms (focal_slab_fast / focal_slab) in place of the SigLIP ones, on the same slab
// geometry and path votes; label sets (as kLabels), ids, groups, top-K lists and the per-sample sums are runtime options.
// kDistill (kModeDistillOpts): the soft-target terms of distillation (distill_slab, the teacher's probabilities in pbuf)
// on the slab geometry and path choice of distill_epilogue, as runtime options everything kFocal takes. Without groups,
// label sets and the per-sample sums, the three sums, g_diag and the sigma operand are those of distill_epilogue bit
// for bit: a slab takes distill_slab<false> or <true> exactly when distill_epilogue does.
template <bool kTopK = false, bool kGroups = false, bool kLabels = false, bool kFocal = false, bool kDistill = false>
__device__ __forceinline__ void sample_loss_epilogue(const KernelParams& p, const float (&acc)[kTileN / 2],
                                                     const CUtensorMap* tmG, uint32_t staging_base, int warp, int wg,
                                                     int lane, int row0, int col_base, int row_lo, int c_lo,
                                                     const Problem& pr, float t_eff, float bias, float tl, float bl,
                                                     uint64_t policy, float& s_sp, float& c_sp, float& s_g, float& c_g,
                                                     float& s_gs, float& c_gs, uint32_t pbuf = 0u) {
  if (p.row_keys != nullptr) tile_metrics(acc, row_lo, col_base, c_lo, pr.M, pr.N, lane, p);
  if constexpr (kTopK) {
    tile_topk(acc, row_lo, col_base, c_lo, pr.M, pr.N, lane, p);
  } else if constexpr (kGroups || kLabels || kFocal || kDistill) {
    if (p.tk_rows != nullptr) tile_topk(acc, row_lo, col_base, c_lo, pr.M, pr.N, lane, p);
  }
  const bool sl = (!kTopK && !kGroups && !kLabels && !kFocal && !kDistill) || p.sl_rows != nullptr;
  // excluded groups: always in kModeGroups, a runtime option in kModeLabels, kModeFocal and kModeDistillOpts
  const bool grp = kGroups || ((kLabels || kFocal || kDistill) && p.col_grp != nullptr);
  // label-set positives: always in kModeLabels, a runtime option in kModeFocal and kModeDistillOpts
  const bool lab = kLabels || ((kFocal || kDistill) && p.col_lab != nullptr);
  // focal: gamma and the weights a_t of the positives and the negatives (both 1 without alpha)
  const float gamma = kFocal ? p.focal_gamma : 0.f;
  const bool alpha = kFocal && p.focal_alpha >= 0.f;
  const float a_pos = alpha ? p.focal_alpha : 1.f, a_neg = alpha ? 1.f - p.focal_alpha : 1.f;
  float acc_sp = 0.f, acc_g = 0.f, acc_gs = 0.f;
  const bool edge = (row0 + kBlockM > pr.M) || (col_base + kTileN > pr.N);
  const bool diag = p.own_chunk && (row0 == col_base);
  const bool sg = p.store_g != 0;
  GStore gst;
  gst.tmap = tmG;
  gst.stage = staging_base + static_cast<uint32_t>(warp) * kStagingBytesPerWarp;
  gst.row0 = row0 + wg * 64 + (warp & 3) * 16;
  gst.lane = lane;
  gst.policy = policy;
  const bool ids = p.row_ids != nullptr, w = p.row_w != nullptr;
  int64_t rid0 = 0, rid1 = 0;
  uint32_t rpos = 0u;
  if (!lab && ids) {   // label sets: the id positives are part of lpos below
    rid0 = p.row_ids[min(row_lo, pr.M - 1)];
    rid1 = p.row_ids[min(row_lo + 8, pr.M - 1)];
    rpos = (row_lo < p.row_pos_n ? 0x3333u : 0u) | (row_lo + 8 < p.row_pos_n ? 0xCCCCu : 0u);
  }
  float rw0 = 1.f, rw1 = 1.f;
  if (w) {
    rw0 = p.row_w[min(row_lo, pr.M - 1)];
    rw1 = p.row_w[min(row_lo + 8, pr.M - 1)];
  }
  int64_t rg0 = -1, rg1 = -1;
  uint32_t rgrp = 0u;   // excl bits of the rows that have a group (>= 0, within grp_rows)
  if ((kGroups || kLabels || kFocal || kDistill) && grp) {
    rg0 = p.row_grp[min(row_lo, p.grp_rows - 1)];
    rg1 = p.row_grp[min(row_lo + 8, p.grp_rows - 1)];
    rgrp = (row_lo < p.grp_rows && rg0 >= 0 ? 0x3333u : 0u) | (row_lo + 8 < p.grp_rows && rg1 >= 0 ? 0xCCCCu : 0u);
  }
  // Label-set positives of the tile's 4 slabs, before the slab loop: the sets of the two fragment rows live in registers
  // only here, next to the accumulator, and the loop carries the 16 pos bits of each slab in one 64-bit word. Rows past
  // M read row M - 1 and columns past N column N - 1: they only lie in edge slabs, which mask them. An empty slot (< 0)
  // and a row slot past lab_m never match, since only column labels >= 0 are compared.
  uint64_t lpos = 0ull;
  if ((kLabels || kFocal || kDistill) && lab) {
    // one fragment row at a time (rows 0 and 8 of the thread's pair) and one slab at a time, not unrolled: one set and
    // one slab's columns are in registers at a time
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      int64_t rl[kMaxLabels];
      const int64_t* rs = p.row_lab + static_cast<size_t>(min(row_lo + 8 * h, pr.M - 1)) * p.lab_m;
#pragma unroll
      for (int k = 0; k < kMaxLabels; ++k) rl[k] = (k < p.lab_m) ? rs[k] : -1;
      // the positional positives of an own chunk whose extras make them id positives (iota ids, own_pos_ids), with the
      // bounds of the ids path
      const bool rid_ok = ids && row_lo + 8 * h < p.row_pos_n;
      const int64_t rid = rid_ok ? p.row_ids[min(row_lo + 8 * h, pr.M - 1)] : 0;
#pragma unroll 1
      for (int c = 0; c < kTileN / 32; ++c) {
        uint32_t lp = 0u;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
          for (int e1 = 0; e1 < 2; ++e1) {
            const int col = col_base + 32 * c + 8 * j + c_lo + e1;
            const int64_t* cs = p.col_lab + static_cast<size_t>(min(col, pr.N - 1)) * p.lab_m;
            bool hit = rid_ok && col < p.col_pos_n && p.col_ids[col] == rid;
#pragma unroll
            for (int k = 0; k < kMaxLabels; ++k) {
              if (k < p.lab_m) {
                const int64_t cl = cs[k];
                if (cl >= 0) {
#pragma unroll
                  for (int q = 0; q < kMaxLabels; ++q) hit |= cl == rl[q];
                }
              }
            }
            lp |= static_cast<uint32_t>(hit) << (4 * j + 2 * h + e1);
          }
        }
        lpos |= static_cast<uint64_t>(lp) << (16 * c);
      }
    }
  }
  float lrow[2] = {0.f, 0.f};
#pragma unroll
  for (int c = 0; c < kTileN / 32; ++c) {
    const float* v = acc + 16 * c;
    const int col0 = col_base + 32 * c;
    float cw[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) cw[j] = w ? p.col_w[min(col0 + 8 * (j >> 1) + c_lo + (j & 1), pr.N - 1)] : 1.f;
    const bool slab_diag = diag && (gst.row0 < col0 + 32) && (col0 < gst.row0 + 16);
    const bool slab_edge = edge && ((gst.row0 + 16 > pr.M) || (col0 + 32 > pr.N));
    uint32_t pos = 0;
    bool slab_pos = false;
    if (!lab && ids) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int e1 = 0; e1 < 2; ++e1) {
          const int col = col0 + 8 * j + c_lo + e1;
          if (col < p.col_pos_n) {
            const int64_t cid = p.col_ids[col];
            pos |= static_cast<uint32_t>(cid == rid0) << (4 * j + e1);
            pos |= static_cast<uint32_t>(cid == rid1) << (4 * j + 2 + e1);
          }
        }
      }
      pos &= rpos;
      slab_pos = __any_sync(0xffffffffu, pos != 0u);
    }
    if ((kLabels || kFocal || kDistill) && lab) {
      pos |= static_cast<uint32_t>(lpos >> (16 * c)) & 0xFFFFu;
      slab_pos = __any_sync(0xffffffffu, pos != 0u);
    }
    uint32_t excl = 0u;
    bool slab_excl = false;
    if ((kGroups || kLabels || kFocal || kDistill) && grp) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int e1 = 0; e1 < 2; ++e1) {
          // a column beyond N reads column N - 1: it only lies in edge slabs, which mask it
          const int64_t cg = p.col_grp[min(col0 + 8 * j + c_lo + e1, pr.N - 1)];
          excl |= static_cast<uint32_t>(cg == rg0) << (4 * j + e1);
          excl |= static_cast<uint32_t>(cg == rg1) << (4 * j + 2 + e1);
        }
      }
      excl &= rgrp & ~pos;   // the own diagonal is tested before excl in loss_slab (slab_diag takes that path anyway)
      slab_excl = __any_sync(0xffffffffu, excl != 0u);
    }
    float lcol[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if constexpr (kDistill) {
      // the series / exact choice is made per slab inside (distill_slab_series)
      if (!slab_edge && !slab_diag && !slab_pos && !slab_excl)
        distill_slab<false, true>(v, pbuf, c, t_eff, bias, tl, bl, p.distill_lambda, row_lo, col0, c_lo, pr.M, pr.N,
                                  sg, gst, p.g_scale, p.g_diag, false, 0u, w, cw, rw0, rw1, acc_sp, acc_g, acc_gs, lrow,
                                  lcol);
      else
        distill_slab<true, true, true>(v, pbuf, c, t_eff, bias, tl, bl, p.distill_lambda, row_lo, col0, c_lo, pr.M,
                                       pr.N, sg, gst, p.g_scale, p.g_diag, slab_diag, pos, w, cw, rw0, rw1, acc_sp,
                                       acc_g, acc_gs, lrow, lcol, excl);
    } else if constexpr (kFocal) {
      // the series path for the slabs the SigLIP kernels send down loss_slab_fast, the general path for all others
      bool fast = false;
      if (!slab_edge && !slab_diag && !slab_pos && !slab_excl) {
        float smax = v[0];
#pragma unroll
        for (int j = 1; j < 16; ++j) smax = fmaxf(smax, v[j]);
        fast = __all_sync(0xffffffffu, fmaf(smax, t_eff, bias) < kFastZ);
      }
      if (fast)
        focal_slab_fast(v, tl, bl, gamma, a_neg, col0, sg, gst, p.g_scale, acc_sp, acc_g, acc_gs, cw, rw0, rw1, lrow,
                        lcol);
      else
        focal_slab(v, t_eff, bias, gamma, a_pos, a_neg, row_lo, col0, c_lo, pr.M, pr.N, sg, gst, p.g_scale, p.g_diag,
                   slab_diag, pos, excl, acc_sp, acc_g, acc_gs, cw, rw0, rw1, lrow, lcol);
    } else if (!slab_edge && !slab_diag && !slab_pos && !slab_excl) {
      float smax = v[0];
#pragma unroll
      for (int j = 1; j < 16; ++j) smax = fmaxf(smax, v[j]);
      const bool fast = __all_sync(0xffffffffu, fmaf(smax, t_eff, bias) < kFastZ);
      if (fast)
        loss_slab_fast<true, true>(v, tl, bl, col0, sg, gst, p.g_scale, acc_sp, acc_g, acc_gs, cw, rw0, rw1, lrow,
                                   lcol);
      else
        loss_slab<false, true, true>(v, t_eff, bias, row_lo, col0, c_lo, pr.M, pr.N, sg, gst, p.g_scale, p.g_diag,
                                     false, 0u, acc_sp, acc_g, acc_gs, cw, rw0, rw1, lrow, lcol);
    } else {
      loss_slab<true, true, true, kGroups || kLabels>(v, t_eff, bias, row_lo, col0, c_lo, pr.M, pr.N, sg, gst,
                                                      p.g_scale, p.g_diag, slab_diag, pos, acc_sp, acc_g, acc_gs, cw,
                                                      rw0, rw1, lrow, lcol, excl);
    }
    if (sl) {
      // reduce-scatter: after the step over lane bit m, lcol[0 .. h) holds the columns q = k + (bit m of lane ? h : 0)
#pragma unroll
      for (int h = 4, m = 16; h >= 1; h >>= 1, m >>= 1) {
        const bool hi = (lane & m) != 0;
#pragma unroll
        for (int k = 0; k < h; ++k) {
          const float send = hi ? lcol[k] : lcol[k + h];
          const float keep = hi ? lcol[k + h] : lcol[k];
          lcol[k] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
      }
      const int q = lane >> 2;
      const int col = col0 + 8 * (q >> 1) + c_lo + (q & 1);
      if (col < pr.N) sample_loss_add(p.sl_cols + col, p.sl_poison, lcol[0]);
    }
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    lrow[0] += __shfl_xor_sync(0xffffffffu, lrow[0], o);
    lrow[1] += __shfl_xor_sync(0xffffffffu, lrow[1], o);
  }
  if (sl && (lane & 3) == 0) {
    if (row_lo < pr.M) sample_loss_add(p.sl_rows + row_lo, p.sl_poison, lrow[0]);
    if (row_lo + 8 < pr.M) sample_loss_add(p.sl_rows + row_lo + 8, p.sl_poison, lrow[1]);
  }
  kahan_add(s_sp, c_sp, acc_sp);
  kahan_add(s_g, c_g, acc_g);
  kahan_add(s_gs, c_gs, acc_gs);
}

// -------------------------------------------------------------------------------------------------
// The kernel
// -------------------------------------------------------------------------------------------------
// kF8: the out kernel of the 8-bit measurement path (its own instantiation: the extra fp32 result registers of
// mma_loop_f8 would otherwise cost the production kernels spills).
// kIds: the loss kernel with labels from sample ids (SIGLIP_OPT_SAMPLE_IDS); its own instantiation, so that the default
// loss kernel is exactly the code it was without the option.
// kMetrics: the loss kernel that also reduces the row / column argmax keys of every tile (siglip_request_metrics); its
// own instantiation for the same reason.
// kWeights: the loss kernel with per-sample weights (SIGLIP_OPT_SAMPLE_WEIGHTS); its own instantiation for the same
// reason, composing with kIds and kMetrics.
// kTileNT: columns of a tile. 256 (kWideTileN) exists for the out kernel with 16-bit operands only (no split-K).
// kMode = kModeDistill: the loss kernel of a distillation step, its own instantiation (kDistillStages, 128-column
// tiles): the teacher's k-blocks of every tile first (tmA1 / tmB1), its probabilities in shared memory, then the
// student's k-loop and the soft-target epilogue (distill_epilogue); ids, weights and metrics are runtime options there.
// kMode = kModeSampleLoss: the loss kernel of a step with per-sample losses, its own instantiation (both stage counts,
// 128-column tiles, K-major operands): the kModeLoss epilogue plus the fixed-point row / column sums
// (sample_loss_epilogue); ids, weights and metrics are runtime options there.
// kMode = kModeTopK: the loss kernel of a top-K step, its own instantiation like kModeSampleLoss: the top-K insertion
// (tile_topk), then the kModeSampleLoss epilogue; ids, weights, metrics and the per-sample-loss sums are runtime options.
// kMode = kModeGroups: the loss kernel of a step that excludes same-group pairs, its own instantiation like
// kModeSampleLoss: its epilogue with the group comparisons (sample_loss_epilogue<false, true>); ids, weights, metrics,
// the per-sample-loss sums and the top-K lists are runtime options.
// kMode = kModeLabels: the loss kernel of a step with label sets, its own instantiation like kModeGroups: its epilogue
// with the set intersections (sample_loss_epilogue<false, false, true>); ids, weights, metrics, the per-sample-loss
// sums, the top-K lists and excluded groups are runtime options.
// kMode = kModeFocal: the loss kernel of a focal step, its own instantiation like kModeLabels: its epilogue with the
// focal terms (sample_loss_epilogue<false, false, false, true>); ids, label sets, weights, metrics, the per-sample-loss
// sums, the top-K lists and excluded groups are runtime options.
// kMode = kModeDistillOpts: the loss kernel of a distillation step with per-sample losses, top-K lists, excluded groups
// or label sets, its own instantiation like kModeDistill: its teacher pass, then the kModeFocal epilogue with the
// soft-target terms (sample_loss_epilogue<false, false, false, false, true>); every option kModeFocal takes is a
// runtime option.
template <int kMode, int kStagesT, int kCS, bool kF8 = false, bool kIds = false, bool kMetrics = false,
          bool kWeights = false, int kTileNT = kTileN>
__global__ void __launch_bounds__(kNumThreads, 1)
siglip_gemm_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmB0,
                   const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB1,
                   const __grid_constant__ CUtensorMap tmG, const __grid_constant__ KernelParams p) {
  using C = Cfg<kMode, kStagesT, kTileNT>;
  static_assert(kCS == 1 || kCS == 2 || kCS == 4, "clusters of 1, 2 or 4 CTAs");
  static_assert(!kIds || kMode == kModeLoss, "sample ids are a loss-kernel option");
  static_assert(!kMetrics || kMode == kModeLoss, "retrieval metrics are a loss-kernel option");
  static_assert(!kWeights || kMode == kModeLoss, "sample weights are a loss-kernel option");
  static_assert(kTileNT == kTileN || (kTileNT == kWideTileN && kMode == kModeOut && !kF8),
                "256-column tiles: out kernel, 16-bit operands");
  static_assert(kMode != kModeDistill || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the distillation kernel takes ids, weights and metrics as runtime options");
  static_assert(kMode != kModeSampleLoss || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the per-sample-loss kernel takes ids, weights and metrics as runtime options");
  static_assert(kMode != kModeTopK || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the top-K kernel takes ids, weights, metrics and per-sample losses as runtime options");
  static_assert(kMode != kModeGroups || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the excluded-groups kernel takes ids, weights, metrics, per-sample losses and top-K as runtime options");
  static_assert(kMode != kModeLabels || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the label-set kernel takes its other options at run time");
  static_assert(kMode != kModeFocal || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the focal kernel takes its other options at run time");
  static_assert(kMode != kModeDistillOpts || (!kF8 && !kIds && !kMetrics && !kWeights && kTileNT == kTileN),
                "the distillation kernel with options takes its other options at run time");
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned stage bases
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t staging_base = smem_base + C::kStages * C::kStageBytes;
  const uint32_t bar_base = staging_base + C::kStagingBytes;
  // barrier map (8 bytes each): full[kStages], empty[kStages], then the loss kernel's reduction slots
  const uint32_t full0 = bar_base, empty0 = bar_base + 8u * C::kStages;
  const uint32_t red_smem = bar_base + 16u * C::kStages;  // 8 warps x 3 doubles

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (p.aux_trace != nullptr && threadIdx.x == 0) {
    const unsigned long long now = globaltimer_ns();
    if (blockIdx.x == 0) p.aux_trace[4] = now;                                       // kernel entry (CTA 0)
    atomicMax(p.aux_trace + 12, now);                                                // ... of the last CTA to start
    atomicMin(p.aux_trace + 13, now);                                                // ... of the first
  }
  const uint32_t crank = (kCS > 1) ? cluster_ctarank() : 0u;
  constexpr uint16_t kMcMask = static_cast<uint16_t>((1u << kCS) - 1u);  // every CTA of the cluster
  const int cluster_id = blockIdx.x / kCS;
  const int num_clusters = gridDim.x / kCS;
  const int whole_tiles = cluster_tiles(p.prob[0]) + (p.nprob > 1 ? cluster_tiles(p.prob[1]) : 0);
  const int total_tiles = (p.sk_parts > 1) ? p.sk_first + p.sk_tiles * p.sk_parts : whole_tiles;

  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmA0);
    prefetch_tmap(&tmB0);
    if (p.nprob > 1) {
      prefetch_tmap(&tmA1);
      prefetch_tmap(&tmB1);
    }
    if constexpr (teacher_mode(kMode)) {
      prefetch_tmap(&tmA1);
      prefetch_tmap(&tmB1);
    }
  }
  if (warp == kInitWarp && lane == 0) {
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(full0 + 8u * s, 1);
      // every consumer warp of every CTA that multicasts into this stage must have released it
      mbar_init(empty0 + 8u * s, kNumEpiWarps * kCS);
    }
    fence_mbar_init();
  }
  if constexpr (kCS > 1) {
    cluster_sync_all();
  } else {
    __syncthreads();
  }
  // Programmatic dependent launch: everything above (barriers, descriptor prefetch) touched no global memory and
  // may run while the previous kernel of the stream drains its last tiles; from here on its results are needed (and the
  // buffers it read are overwritten). The next kernel of the stream may start ITS set-up as soon as SMs free up.
  if (p.pdl) {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  }
  if (p.aux_trace != nullptr && threadIdx.x == 0) {
    const unsigned long long now = globaltimer_ns();
    if (blockIdx.x == 0) p.aux_trace[5] = now;                                       // set-up done (CTA 0)
    atomicMax(p.aux_trace + 14, now);                                                // ... on the last CTA
  }

  if (warp == kProducerWarp) {
    // ===================================== TMA producer =====================================
    // The whole warp runs the loop (warp-uniform control flow); one elected lane issues the TMA instructions.
    int stage = 0;
    uint32_t phase = 0;
    long long w_empty = 0;
    // L2 priorities: the embeddings (A and B of the loss kernel, B of the gradient kernel) are re-read by every tile
    // wave and must survive the sigma operand streaming through the 50 MB L2 once per pass. The sigma operand itself
    // keeps normal priority: the column tiles of a row panel read the same lines a little apart in time.
    const uint64_t pol_b = l2_policy_evict_last();
    const uint64_t pol_a = (kMode != kModeOut) ? pol_b : l2_policy_evict_normal();
    for (int t = cluster_id; t < total_tiles; t += num_clusters) {
      const TileCoord tc = decode_tile<kCS>(p, t, static_cast<int>(crank));
      const Problem& pr = p.prob[tc.prob];
      const CUtensorMap* tmA = tc.prob ? &tmA1 : &tmA0;
      const CUtensorMap* tmB = tc.prob ? &tmB1 : &tmB0;
      const int m_idx = tc.m_blk * kBlockM;
      const int n_idx = tc.n_blk * kTileNT;
      // elements per 128-byte swizzle row: 64 16-bit values, or 128 8-bit ones (fp8 measurement path, K-major only)
      const int kblk = (pr.ab_f16 == 2) ? 2 * kBlockK : kBlockK;
      const int num_kb = (pr.K + kblk - 1) / kblk;
      const int a_mn = pr.a_mn, b_mn = pr.b_mn;
      int kb0, kb1;
      item_k_range(p, tc, num_kb, kb0, kb1);
      if constexpr (teacher_mode(kMode)) {
        // the teacher's k-blocks of the tile first (both K-major, K = D_T), through the same ring
        constexpr int kRows = kTileN / kCS;
        const int num_kb_t = (p.k_teacher + kBlockK - 1) / kBlockK;
        for (int kb = 0; kb < num_kb_t; ++kb) {
          mbar_wait(empty0 + 8u * stage, phase ^ 1u, p.dbg, 1, t, kb, 0, p.wait_stats ? &w_empty : nullptr);
          if (elect_one_sync()) {
            const uint32_t sA = smem_base + stage * C::kStageBytes;
            const uint32_t sB = sA + C::kABytes;
            const uint32_t fb = full0 + 8u * stage;
            mbar_arrive_expect_tx(fb, C::kStageBytes);
            tma_load_2d_hint(&tmA1, fb, sA, kb * kBlockK, m_idx, pol_a);
            const uint32_t dst = sB + crank * (kRows * 128);
            if constexpr (kCS == 1)
              tma_load_2d_hint(&tmB1, fb, dst, kb * kBlockK, n_idx, pol_b);
            else
              tma_load_2d_mcast(&tmB1, fb, dst, kb * kBlockK, n_idx + static_cast<int>(crank) * kRows, kMcMask);
          }
          __syncwarp();
          if (++stage == C::kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(empty0 + 8u * stage, phase ^ 1u, p.dbg, 1, t, kb, 0, p.wait_stats ? &w_empty : nullptr);
        if (elect_one_sync()) {
          const uint32_t sA = smem_base + stage * C::kStageBytes;
          const uint32_t sB = sA + C::kABytes;
          const uint32_t fb = full0 + 8u * stage;
          // A of this CTA plus the WHOLE B tile: the other CTAs of the cluster multicast their shares into it
          mbar_arrive_expect_tx(fb, C::kStageBytes);
          const int k_idx = kb * kblk;
          if (!a_mn) {
            tma_load_2d_hint(tmA, fb, sA, k_idx, m_idx, pol_a);    // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int h = 0; h < kBlockM / 64; ++h)                  // boxes {64 rows, 64 k}
              tma_load_2d_hint(tmA, fb, sA + h * 8192, m_idx + 64 * h, k_idx, pol_a);
          }
          // this CTA's 1 / kCS of the B tile, delivered to every CTA of the cluster
          auto load_b = [&](uint32_t dst, int c0, int c1) {
            if constexpr (kCS == 1) {
              tma_load_2d_hint(tmB, fb, dst, c0, c1, pol_b);
            } else {
              tma_load_2d_mcast(tmB, fb, dst, c0, c1, kMcMask);
            }
          };
          if (!b_mn) {
            constexpr int kRows = kTileNT / kCS;                    // box {64 k, kRows rows}
            load_b(sB + crank * (kRows * 128), k_idx, n_idx + static_cast<int>(crank) * kRows);
          } else if constexpr (kCS == 4 && kTileNT == kTileN) {
            // boxes {64 columns, 32 k}: CTA r fetches k half (r & 1) of the 64-column block (r >> 1)
            const int h = static_cast<int>(crank >> 1), kh = static_cast<int>(crank & 1u);
            load_b(sB + h * 8192 + kh * 4096, n_idx + 64 * h, k_idx + 32 * kh);
          } else {
            constexpr int kBoxes = kTileNT / 64;                    // boxes {64 columns, 64 k}, kBoxes / kCS per CTA
#pragma unroll
            for (int h = static_cast<int>(crank) * (kBoxes / kCS); h < (static_cast<int>(crank) + 1) * (kBoxes / kCS); ++h)
              load_b(sB + h * 8192, n_idx + 64 * h, k_idx);
          }
        }
        __syncwarp();
        if (++stage == C::kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
    if (p.wait_stats && lane == 0) p.wait_stats[8ll * blockIdx.x + 0] = static_cast<unsigned long long>(w_empty);
  } else if (warp < kNumEpiWarps) {
    // ===================================== consumers: MMA + epilogue =====================================
    const int wg = warp >> 2;                       // warpgroup: rows [64 wg, 64 wg + 64) of the CTA's block
    const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // first fragment row (the second is r_lo + 8)
    const int c_lo = 2 * (lane & 3);                // first fragment column of every 8-column group
    const float t_exact = expf(load_t_prime(p));
    const float bias = (kMode != kModeOut) ? *p.bias : 0.f;
    // loss kernel: z = t_eff * acc + b with t_eff = t * s_scale (the accumulator is 2^8 <img, txt> for fp16 x 16 operands)
    const float s_scale = (kMode != kModeOut && p.s_scale != 0.f) ? p.s_scale : 1.0f;
    const float t_eff = t_exact * s_scale;
    const float tl = t_eff * kLog2e, bl = bias * kLog2e;
    // distillation: the teacher's z^T = t_T s^T + b_T (its accumulator is 2^8 s^T for fp16 x 16 operands)
    float tT_eff = 0.f, bias_T = 0.f, tT_l = 0.f, bT_l = 0.f;
    uint32_t pbuf = 0;
    if constexpr (teacher_mode(kMode)) {
      tT_eff = expf(*p.t_prime_T) * (p.teacher_f16 ? 1.0f / 256.0f : 1.0f);
      bias_T = *p.bias_T;
      tT_l = tT_eff * kLog2e;
      bT_l = bias_T * kLog2e;
      pbuf = bar_base + 1024u;   // behind the barrier block (Cfg::kPBytes)
    }
    // per-thread running sums over the tiles of this CTA: compensated fp32 (Kahan); fp64 only at the very end
    float s_sp = 0.f, s_g = 0.f, s_gs = 0.f, c_sp = 0.f, c_g = 0.f, c_gs = 0.f;
    long long w_full = 0;
    long long* w_full_p = (p.wait_stats != nullptr && threadIdx.x == 0) ? &w_full : nullptr;
    if constexpr (kMode == kModeOut) {
      // backward of the two scalars: saved (upstream gradient 1) * grad_out, by one thread of the launch
      if (blockIdx.x == 0 && threadIdx.x == 0 && p.sc_saved != nullptr) {
        const float g = (p.grad_out != nullptr) ? *p.grad_out : 1.0f;
        if (p.sc_dt_prime) {
          if (p.tprime_f64)
            *reinterpret_cast<double*>(p.sc_dt_prime) = static_cast<double>(p.sc_saved[0] * g);
          else
            *p.sc_dt_prime = p.sc_saved[0] * g;
        }
        if (p.sc_dbias) *p.sc_dbias = p.sc_saved[1] * g;
      }
    }
    const uint64_t g_store_policy = l2_policy_evict_first();
    const long long c_start = clock_cycles();
    int stage = 0;
    uint32_t phase = 0;
    bool p1_ready = false;
    float acc[kTileNT / 2];
    float acc8[kF8 ? 64 : 1];   // result of the 8-bit mainloop (see mma_loop_f8)
    for (int t = cluster_id; t < total_tiles; t += num_clusters) {
      const TileCoord tc = decode_tile<kCS>(p, t, static_cast<int>(crank));
      const Problem& pr = p.prob[tc.prob];
      const int row0 = tc.m_blk * kBlockM;            // first row of this CTA's block
      const int col_base = tc.n_blk * kTileNT;
      const int row_lo = row0 + r_lo;                 // global rows of this thread: row_lo, row_lo + 8
      const bool fp8 = (pr.ab_f16 == 2);
      const int num_kb = (pr.K + (fp8 ? 2 * kBlockK : kBlockK) - 1) / (fp8 ? 2 * kBlockK : kBlockK);
      int kb0, kb1;
      item_k_range(p, tc, num_kb, kb0, kb1);
      {
        // K-major: 8-row groups 1024 B apart (SBO), K advance 32 B inside the swizzle row (16 16-bit or 32 8-bit values).
        // MN-major: 64-element MN blocks 8192 B apart (LBO), 8-k groups 1024 B apart (SBO), K advance 16 rows.
        // This warpgroup's 64 A rows start 8192 B into the A tile in both layouts. A 256-column MN-major B tile is 4
        // such 64-column blocks (the same LBO), a K-major one 256 rows of 8-row groups (the same SBO).
        const uint32_t a_lbo = pr.a_mn ? 8192u : 16u, b_lbo = pr.b_mn ? 8192u : 16u;
        const uint32_t a_adv = pr.a_mn ? (kMmaK * 128u) >> 4 : 32u >> 4;
        const uint32_t b_adv = pr.b_mn ? (kMmaK * 128u) >> 4 : 32u >> 4;
        const uint64_t adesc0 = make_smem_desc_sw128(smem_base + static_cast<uint32_t>(wg) * 8192u, a_lbo, 1024u);
        const uint64_t bdesc0 = make_smem_desc_sw128(smem_base + C::kABytes, b_lbo, 1024u);
        if constexpr (teacher_mode(kMode)) {
          // s^T of the tile over the teacher's k-blocks, then p = sigma(t_T s^T + b_T) into this thread's slots. The
          // student's k-loop below starts from zero (its first wgmma does not accumulate); the producer is already
          // streaming its operands while the conversion runs.
          const int num_kb_t = (p.k_teacher + kBlockK - 1) / kBlockK;
          if (p.teacher_f16)
            mma_loop<1, 0, 0, kCS, C::kStageBytes, kTileN>(acc, 0, num_kb_t, stage, phase, C::kStages, adesc0, bdesc0,
                                                           a_adv, b_adv, full0, empty0, lane, p.dbg, t, w_full_p);
          else
            mma_loop<0, 0, 0, kCS, C::kStageBytes, kTileN>(acc, 0, num_kb_t, stage, phase, C::kStages, adesc0, bdesc0,
                                                           a_adv, b_adv, full0, empty0, lane, p.dbg, t, w_full_p);
#pragma unroll
          for (int c = 0; c < kTileN / 32; ++c) {
            const bool series = distill_slab_series(acc + 16 * c, tT_eff, bias_T);
#pragma unroll
            for (int i = 16 * c; i < 16 * c + 16; ++i) {
              const float pv = distill_sigma(acc[i], tT_eff, bias_T, tT_l, bT_l, series);
              asm volatile("st.shared.f32 [%0], %1;" ::"r"(distill_p_addr(pbuf, i)), "f"(pv) : "memory");
            }
          }
        }
#define SIGLIP_MMA_LOOP(T, TA, TB)                                                                                  \
  mma_loop<T, TA, TB, kCS, C::kStageBytes, kTileNT>(acc, kb0, kb1, stage, phase, C::kStages, adesc0, bdesc0, a_adv, \
                                                    b_adv, full0, empty0, lane, p.dbg, t, w_full_p)
        const int sel = pr.a_mn * 2 + pr.b_mn;
        if constexpr (teacher_mode(kMode) || kMode == kModeSampleLoss || kMode == kModeTopK || kMode == kModeGroups ||
                      kMode == kModeLabels || kMode == kModeFocal) {
          // the loss operands (student and teacher) are always K-major: no MN-major variants in this instantiation
          if (pr.ab_f16)
            SIGLIP_MMA_LOOP(1, 0, 0);
          else
            SIGLIP_MMA_LOOP(0, 0, 0);
        } else if (fp8) {
          // kF8 instantiation only (launch_gemm routes 8-bit operands there): the result lands in acc8
          if constexpr (kF8)
            mma_loop_f8<kCS, C::kStageBytes>(acc8, acc, kb0, kb1, stage, phase, C::kStages, adesc0, bdesc0, full0,
                                             empty0, lane, p.dbg, t, w_full_p);
        } else if (pr.ab_f16) {
          switch (sel) {
            case 0: SIGLIP_MMA_LOOP(1, 0, 0); break;
            case 1: SIGLIP_MMA_LOOP(1, 0, 1); break;
            case 2: SIGLIP_MMA_LOOP(1, 1, 0); break;
            default: SIGLIP_MMA_LOOP(1, 1, 1); break;
          }
        } else {
          switch (sel) {
            case 0: SIGLIP_MMA_LOOP(0, 0, 0); break;
            case 1: SIGLIP_MMA_LOOP(0, 0, 1); break;
            case 2: SIGLIP_MMA_LOOP(0, 1, 0); break;
            default: SIGLIP_MMA_LOOP(0, 1, 1); break;
          }
        }
#undef SIGLIP_MMA_LOOP
      }
      if (p.aux_trace != nullptr && threadIdx.x == 0 && t == cluster_id && blockIdx.x == 0)
        p.aux_trace[6] = globaltimer_ns();                                   // first tile's MMAs done (CTA 0)

      if constexpr (kMode == kModeDistill) {
        distill_epilogue(p, acc, pbuf, &tmG, staging_base, warp, wg, lane, row0, col_base, row_lo, c_lo, pr, t_eff, bias,
                         tl, bl, g_store_policy, s_sp, c_sp, s_g, c_g, s_gs, c_gs);
      } else if constexpr (kMode == kModeSampleLoss) {
        sample_loss_epilogue(p, acc, &tmG, staging_base, warp, wg, lane, row0, col_base, row_lo, c_lo, pr, t_eff, bias,
                             tl, bl, g_store_policy, s_sp, c_sp, s_g, c_g, s_gs, c_gs);
      } else if constexpr (kMode == kModeTopK) {
        sample_loss_epilogue<true>(p, acc, &tmG, staging_base, warp, wg, lane, row0, col_base, row_lo, c_lo, pr, t_eff,
                                   bias, tl, bl, g_store_policy, s_sp, c_sp, s_g, c_g, s_gs, c_gs);
      } else if constexpr (kMode == kModeGroups) {
        sample_loss_epilogue<false, true>(p, acc, &tmG, staging_base, warp, wg, lane, row0, col_base, row_lo, c_lo, pr,
                                          t_eff, bias, tl, bl, g_store_policy, s_sp, c_sp, s_g, c_g, s_gs, c_gs);
      } else if constexpr (kMode == kModeLabels) {
        sample_loss_epilogue<false, false, true>(p, acc, &tmG, staging_base, warp, wg, lane, row0, col_base, row_lo,
                                                 c_lo, pr, t_eff, bias, tl, bl, g_store_policy, s_sp, c_sp, s_g, c_g,
                                                 s_gs, c_gs);
      } else if constexpr (kMode == kModeFocal) {
        sample_loss_epilogue<false, false, false, true>(p, acc, &tmG, staging_base, warp, wg, lane, row0, col_base,
                                                        row_lo, c_lo, pr, t_eff, bias, tl, bl, g_store_policy, s_sp,
                                                        c_sp, s_g, c_g, s_gs, c_gs);
      } else if constexpr (kMode == kModeDistillOpts) {
        sample_loss_epilogue<false, false, false, false, true>(p, acc, &tmG, staging_base, warp, wg, lane, row0,
                                                               col_base, row_lo, c_lo, pr, t_eff, bias, tl, bl,
                                                               g_store_policy, s_sp, c_sp, s_g, c_g, s_gs, c_gs, pbuf);
      } else if constexpr (kMode == kModeLoss) {
        // argmax keys first, on the raw accumulator: whichever path each slab then takes below
        if constexpr (kMetrics) tile_metrics(acc, row_lo, col_base, c_lo, pr.M, pr.N, lane, p);
        float acc_sp = 0.f, acc_g = 0.f, acc_gs = 0.f;
        const bool edge = (row0 + kBlockM > pr.M) || (col_base + kTileN > pr.N);
        // 128-aligned row and column blocks: only a block on the diagonal holds positive pairs
        const bool diag = p.own_chunk && (row0 == col_base);
        const bool sg = p.store_g != 0;
        GStore gst;
        gst.tmap = &tmG;
        gst.stage = staging_base + static_cast<uint32_t>(warp) * kStagingBytesPerWarp;
        gst.row0 = row0 + wg * 64 + (warp & 3) * 16;
        gst.lane = lane;
        gst.policy = g_store_policy;
        // Sample-id labels (kIds): the ids of this thread's two fragment rows, loaded once per tile (a row beyond M takes
        // row M - 1's id: it only lies in edge slabs, which mask it).
        int64_t rid0 = 0, rid1 = 0;
        uint32_t rpos = 0u;   // pos bits of the rows that carry ids: an extra image past row_pos_n never matches
        if constexpr (kIds) {
          rid0 = p.row_ids[min(row_lo, pr.M - 1)];
          rid1 = p.row_ids[min(row_lo + 8, pr.M - 1)];
          rpos = (row_lo < p.row_pos_n ? 0x3333u : 0u) | (row_lo + 8 < p.row_pos_n ? 0xCCCCu : 0u);
        }
        // Sample weights (kWeights): the weights of the two fragment rows, once per tile (clamped like the ids)
        float rw0 = 1.f, rw1 = 1.f;
        if constexpr (kWeights) {
          rw0 = p.row_w[min(row_lo, pr.M - 1)];
          rw1 = p.row_w[min(row_lo + 8, pr.M - 1)];
        }
#pragma unroll
        for (int c = 0; c < kTileN / 32; ++c) {
          const float* v = acc + 16 * c;
          const int col0 = col_base + 32 * c;
          // kWeights: the slab's 8 column weights of this thread, cw[2 j + e1] for column 8 j + c_lo + e1 (a column
          // beyond N reads column N - 1: it only lies in edge slabs, which mask it)
          float cw[kWeights ? 8 : 1];
          if constexpr (kWeights) {
#pragma unroll
            for (int j = 0; j < 8; ++j) cw[j] = p.col_w[min(col0 + 8 * (j >> 1) + c_lo + (j & 1), pr.N - 1)];
          }
          // Only the 16x32 slabs that touch the diagonal of a diagonal block hold positive pairs, and only the slabs
          // that cross the matrix border of an edge block need masking; every other slab takes the fast path like
          // the rest of the matrix.
          const bool slab_diag = diag && (gst.row0 < col0 + 32) && (col0 < gst.row0 + 16);
          const bool slab_edge = edge && ((gst.row0 + 16 > pr.M) || (col0 + 32 > pr.N));
          // With sample ids, a slab in which any element's ids match (slab_pos) also takes the label-applying path.
          // pos bit i <-> fragment element i (row r_lo + 8 ((i >> 1) & 1), column 8 (i >> 2) + c_lo + (i & 1)).
          uint32_t pos = 0;
          bool slab_pos = false;
          if constexpr (kIds) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
              for (int e1 = 0; e1 < 2; ++e1) {
                const int col = col0 + 8 * j + c_lo + e1;
                if (col < p.col_pos_n) {   // texts with ids only: a hard negative has none and is never positive
                  const int64_t cid = p.col_ids[col];
                  pos |= static_cast<uint32_t>(cid == rid0) << (4 * j + e1);
                  pos |= static_cast<uint32_t>(cid == rid1) << (4 * j + 2 + e1);
                }
              }
            }
            pos &= rpos;
            slab_pos = __any_sync(0xffffffffu, pos != 0u);
          }
          if (!slab_edge && !slab_diag && !slab_pos) {
            // z is monotone in s (t > 0): the slab is "all very negative" iff max s is
            float smax = v[0];
#pragma unroll
            for (int j = 1; j < 16; ++j) smax = fmaxf(smax, v[j]);
            const bool fast = __all_sync(0xffffffffu, fmaf(smax, t_eff, bias) < kFastZ);
            if (fast)
              loss_slab_fast<kWeights>(v, tl, bl, col0, sg, gst, p.g_scale, acc_sp, acc_g, acc_gs, cw, rw0, rw1);
            else
              loss_slab<false, kWeights>(v, t_eff, bias, row_lo, col0, c_lo, pr.M, pr.N, sg, gst, p.g_scale, p.g_diag,
                                         false, 0u, acc_sp, acc_g, acc_gs, cw, rw0, rw1);
          } else {
            loss_slab<true, kWeights>(v, t_eff, bias, row_lo, col0, c_lo, pr.M, pr.N, sg, gst, p.g_scale, p.g_diag,
                                      slab_diag, pos, acc_sp, acc_g, acc_gs, cw, rw0, rw1);
          }
        }
        kahan_add(s_sp, c_sp, acc_sp);
        kahan_add(s_g, c_g, acc_g);
        kahan_add(s_gs, c_gs, acc_gs);
      } else {
        const float scale = t_exact * p.inv_b * (p.grad_out != nullptr ? *p.grad_out : 1.0f);
        // the positive-pair term exists for the first fix_rows rows only (the dtxt problem of an own chunk with hard
        // negatives has M = T rows, but fix_vec / fix_mat hold this rank's B)
        const float fix0 = (pr.fix_vec != nullptr && row_lo < p.fix_rows) ? pr.fix_vec[row_lo] : 0.f;
        const float fix1 = (pr.fix_vec != nullptr && row_lo + 8 < p.fix_rows) ? pr.fix_vec[row_lo + 8] : 0.f;
        if (tc.prob == 1 && p.p1_wait_flag != nullptr && !p1_ready) {
          // the dtxt tiles of the LAST gradient launch add the folded sum of the peers' contributions: the fold that
          // completes it runs in this very launch (auxiliary warps of all CTAs) and must have finished everywhere
          if (lane == 0) {
            uint64_t t0 = 0;
            uint32_t spins = 0;
            while (true) {
              unsigned int v;
              asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.p1_wait_flag) : "memory");
              if (v >= p.p1_wait_value) break;
              __nanosleep(500);
              if ((++spins & 0xffu) == 0) {
                const uint64_t now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                if (now - t0 > p.peer_timeout_ns) {
                  if (p.dbg != nullptr) {
                    p.dbg->block = blockIdx.x;
                    p.dbg->thread = threadIdx.x;
                    p.dbg->aux0 = v;
                    p.dbg->aux1 = p.p1_wait_value;
                    p.dbg->code = 8;
                    __threadfence_system();
                  }
                  __trap();
                }
              }
            }
          }
          __syncwarp();
          p1_ready = true;
        }
        if constexpr (kF8) {   // whole tiles only: split-K is never requested for 8-bit operands
          out_row<kTileN>(acc8, 0, scale, row_lo, col_base, c_lo, pr, fix0, p.fix_rows);
          out_row<kTileN>(acc8, 1, scale, row_lo + 8, col_base, c_lo, pr, fix1, p.fix_rows);
        } else if (tc.part < 0) {
          out_row<kTileNT>(acc, 0, scale, row_lo, col_base, c_lo, pr, fix0, p.fix_rows);
          out_row<kTileNT>(acc, 1, scale, row_lo + 8, col_base, c_lo, pr, fix1, p.fix_rows);
        } else if constexpr (kTileNT == kTileN) {   // launch_impl splits 128-column tiles only
          // split tile: this CTA's 128 x 128 fp32 partial in fragment order, thread-contiguous float4's
          const size_t kPartF4 = static_cast<size_t>(kBlockM) * kTileN / 4;
          float4* ws = reinterpret_cast<float4*>(p.sk_ws) +
                       (static_cast<size_t>(tc.slot) * (p.sk_parts - 1) * kCS + crank) * kPartF4 + threadIdx.x;
          const size_t part_stride = static_cast<size_t>(kCS) * kPartF4;   // float4 per slice
          if (tc.part > 0) {
            float4* dst = ws + static_cast<size_t>(tc.part - 1) * part_stride;
#pragma unroll
            for (int j4 = 0; j4 < 16; ++j4)
              dst[j4 * (kNumEpiWarps * 32)] = make_float4(acc[4 * j4], acc[4 * j4 + 1], acc[4 * j4 + 2], acc[4 * j4 + 3]);
            // my share of the partial accumulator is written: arrive (release) on the tile's counter
            __threadfence();
            __syncwarp();
            if (lane == 0) atomicAdd(p.sk_counters + 2 * tc.slot, 1u);
          } else {
            // owner slice: the other slices' partial accumulators must be in the workspace (they run at the same time
            // on other clusters and wait for nothing, so this cannot deadlock on a co-resident persistent grid)
            if (lane == 0) {
              const unsigned int need = static_cast<unsigned int>((p.sk_parts - 1) * kCS * kNumEpiWarps);
              const unsigned int* ctr = p.sk_counters + 2 * tc.slot;
              uint64_t t0 = 0;
              uint32_t spins = 0;
              while (true) {
                unsigned int cv;
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cv) : "l"(ctr) : "memory");
                if (cv >= need) break;
                __nanosleep(100);
                if ((++spins & 0x3ffu) == 0) {
                  const uint64_t now = globaltimer_ns();
                  if (t0 == 0) t0 = now;
                  if (now - t0 > SIGLIP_WAIT_TIMEOUT_NS) {
                    if (p.dbg != nullptr) {
                      p.dbg->block = blockIdx.x;
                      p.dbg->thread = threadIdx.x;
                      p.dbg->aux0 = cv;
                      p.dbg->aux1 = need;
                      p.dbg->code = 4;
                      __threadfence_system();
                    }
                    __trap();
                  }
                }
              }
            }
            __syncwarp();
            out_row<kTileN>(acc, 0, scale, row_lo, col_base, c_lo, pr, fix0, p.fix_rows, ws, p.sk_parts - 1,
                            part_stride);
            out_row<kTileN>(acc, 1, scale, row_lo + 8, col_base, c_lo, pr, fix1, p.fix_rows, ws, p.sk_parts - 1,
                            part_stride);
            // every owner warp has consumed the partials: the last one re-arms the counters for the next launch
            __syncwarp();
            if (lane == 0) {
              const unsigned int seen = atomicAdd(p.sk_counters + 2 * tc.slot + 1, 1u);
              if (seen == static_cast<unsigned int>(kCS * kNumEpiWarps) - 1u) {
                p.sk_counters[2 * tc.slot] = 0u;
                p.sk_counters[2 * tc.slot + 1] = 0u;
              }
            }
          }
        }
      }
    }
    if (p.aux_trace != nullptr && threadIdx.x == 0) {
      const unsigned long long now = globaltimer_ns();
      if (blockIdx.x == 0) p.aux_trace[7] = now;                    // last tile done (CTA 0)
      atomicMax(p.aux_trace + 9, now);                              // ... latest / earliest over the CTAs
      atomicMin(p.aux_trace + 10, now);
      atomicMax(p.aux_trace + 11, now);
    }
    if (p.wait_stats != nullptr && threadIdx.x == 0) {
      p.wait_stats[8ll * blockIdx.x + 1] = static_cast<unsigned long long>(w_full);
      p.wait_stats[8ll * blockIdx.x + 3] = static_cast<unsigned long long>(clock_cycles() - c_start);
    }
    if constexpr (kMode != kModeOut) {
      // all sigma slabs of this warp must be in global memory before the kernel ends
      if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
      // fixed-order reduction: lanes -> warp -> consumer warps -> one slot per CTA (summed later in slot order)
      double d_sp = warp_sum(static_cast<double>(s_sp) - static_cast<double>(c_sp));
      double d_g = warp_sum(static_cast<double>(s_g) - static_cast<double>(c_g));
      // sum g * acc -> sum g * <img, txt>
      double d_gs = warp_sum(static_cast<double>(s_gs) - static_cast<double>(c_gs)) * static_cast<double>(s_scale);
      double* red = reinterpret_cast<double*>(smem_raw + (red_smem - smem_u32(smem_raw)));
      if (lane == 0) {
        red[warp * 3 + 0] = d_sp;
        red[warp * 3 + 1] = d_g;
        red[warp * 3 + 2] = d_gs;
      }
      named_barrier_sync(1, kNumEpiWarps * 32);
      if (warp == 0) {
        unsigned int ticket = 0;
        // 8 warps x 3 sums: lanes 0..7 take one warp's triple each, fixed shuffle tree (same order every run)
        double s0 = (lane < kNumEpiWarps) ? red[lane * 3 + 0] : 0.0;
        double s1 = (lane < kNumEpiWarps) ? red[lane * 3 + 1] : 0.0;
        double s2 = (lane < kNumEpiWarps) ? red[lane * 3 + 2] : 0.0;
        s0 = warp_sum(s0);
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        if (lane == 0) {
          double* slot = p.partials + 4ll * blockIdx.x;
          if (p.accumulate_partials) {
            s0 += slot[0];
            s1 += slot[1];
            s2 += slot[2];
          }
          slot[0] = s0;
          slot[1] = s1;
          slot[2] = s2;
          if (p.fin_counter != nullptr) {
            __threadfence();                              // the slot before the ticket
            ticket = atomicAdd(p.fin_counter, 1u);
          }
        }
        if (p.fin_counter != nullptr) {
          ticket = __shfl_sync(0xffffffffu, ticket, 0);
          if (ticket == gridDim.x - 1) {
            // last CTA of the forward's last loss kernel: every slot is final. One warp, slot order and a fixed
            // shuffle tree => bitwise reproducible for a fixed grid
            __threadfence();
            double f0 = 0.0, f1 = 0.0, f2 = 0.0;
            for (unsigned int i = lane; i < gridDim.x; i += 32) {
              f0 += __ldcg(p.partials + 4ll * i + 0);
              f1 += __ldcg(p.partials + 4ll * i + 1);
              f2 += __ldcg(p.partials + 4ll * i + 2);
            }
            f0 = warp_sum(f0);
            f1 = warp_sum(f1);
            f2 = warp_sum(f2);
            if (lane == 0) {
              const double inv_b = static_cast<double>(p.inv_b);
              if (p.fin_loss) *p.fin_loss = static_cast<float>(f0 * inv_b);
              if (p.fin_dbias) *p.fin_dbias = static_cast<float>(f1 * inv_b);
              if (p.fin_dt_prime)
                *p.fin_dt_prime = static_cast<float>(static_cast<double>(expf(load_t_prime(p))) * f2 * inv_b);
              *p.fin_counter = 0u;                        // ready for the next forward
            }
          }
        }
      }
    }
  } else if (warp >= kAuxWarp) {
    // ===================== the two auxiliary warps: NVSwitch peer pull, conversions, fold =====================
    // A text chunk is read ONCE from its owner's buffer (P2P over NVLink) into local HBM while the previous chunk's
    // tiles compute (replaces distributed_utils.py:10-27 neighbour_exchange / the all_gather at
    // distributed_sigmoid_loss.py:35); MMA operands are then fed from local memory only. The peers' dtxt
    // contributions are folded into a local fp32 accumulator the same way (the reduce-scatter of all_gather's backward,
    // torch functional.py:343-354, spread over the steps instead of exposed at the end). Buffer hand-over between the
    // ranks is by flags: waits before a job, release-stores once every CTA has finished its share of it.
    const int aux_tid = static_cast<int>(threadIdx.x) - kAuxWarp * 32;
    const unsigned long long nthreads = static_cast<unsigned long long>(gridDim.x) * 64ull;
    const unsigned long long tid0 = static_cast<unsigned long long>(blockIdx.x) * 64ull + aux_tid;
    const bool tracer = (p.aux_trace != nullptr && blockIdx.x == 0 && aux_tid == 0);
    if (tracer) p.aux_trace[0] = globaltimer_ns();
    unsigned long long waited_until = 0;
#pragma unroll 1
    for (int j = 0; j < p.naux; ++j) {
      const AuxJob& job = p.aux[j];
      if (job.kind == kAuxNone) continue;
      if (job.wait_flags != nullptr) {
        wait_peer_flags(job.wait_flags, job.wait_n, job.wait_value, p.peer_timeout_ns, p.dbg, job.site);
        if (tracer) waited_until = globaltimer_ns();
      }
      const unsigned long long n16 = job.n16;
      if (job.kind == kAuxCopy) {
        // 8 independent 16-byte loads in flight per thread (~1.2 MB per GPU) to cover the NVLink round trip
        unsigned long long i = tid0;
        for (; i + 7ull * nthreads < n16; i += 8ull * nthreads) {
          uint4 v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = ld_peer_16(job.src + i + u * nthreads);
#pragma unroll
          for (int u = 0; u < 8; ++u) job.dst[i + u * nthreads] = v[u];
        }
        for (; i < n16; i += nthreads) job.dst[i] = ld_peer_16(job.src + i);
      } else if (job.kind == kAuxCvt) {
        // bf16 -> scaled fp16 copies of the embeddings for the gradient kernel (its sigma operand is fp16, and an
        // MMA cannot mix fp16 with bf16): done here, off the critical path, while the tiles of this chunk compute.
        const float sc = p.cvt_scale;
        const bool plain = job.cvt_copy != 0;
        auto cvt = [&](uint4 v) {
          if (plain) return v;
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
          uint32_t o[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            o[q] = pack_f16x2_scaled(__uint_as_float(w[q] << 16), __uint_as_float(w[q] & 0xffff0000u), sc);
          }
          return make_uint4(o[0], o[1], o[2], o[3]);
        };
        // 8 independent 16-byte loads in flight per thread: with one the loop was latency-bound (0.26 ms for the two
        // 32 MiB operands of the headline shape, most of the loss kernel's duration, for 128 MiB of traffic)
        unsigned long long i = tid0;
        for (; i + 7ull * nthreads < n16; i += 8ull * nthreads) {
          uint4 v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = ld_peer_16(job.src + i + u * nthreads);
#pragma unroll
          for (int u = 0; u < 8; ++u) job.dst[i + u * nthreads] = cvt(v[u]);
        }
        for (; i < n16; i += nthreads) job.dst[i] = cvt(ld_peer_16(job.src + i));
      } else if (job.kind == kAuxFold) {
        const bool has_in = job.src2 != nullptr;   // first contribution of a backward pass: plain copy
        const float4* acc_in = reinterpret_cast<const float4*>(job.src2);
        float4* acc_out = reinterpret_cast<float4*>(job.dst);
        unsigned long long i = tid0;
        for (; i + 7ull * nthreads < n16; i += 8ull * nthreads) {
          uint4 rv[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) rv[u] = ld_peer_16(job.src + i + u * nthreads);
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            float4 a = has_in ? acc_in[i + u * nthreads] : make_float4(0.f, 0.f, 0.f, 0.f);
            a.x += __uint_as_float(rv[u].x);
            a.y += __uint_as_float(rv[u].y);
            a.z += __uint_as_float(rv[u].z);
            a.w += __uint_as_float(rv[u].w);
            acc_out[i + u * nthreads] = a;
          }
        }
        for (; i < n16; i += nthreads) {
          const uint4 rr = ld_peer_16(job.src + i);
          float4 a = has_in ? acc_in[i] : make_float4(0.f, 0.f, 0.f, 0.f);
          a.x += __uint_as_float(rr.x);
          a.y += __uint_as_float(rr.y);
          a.z += __uint_as_float(rr.z);
          a.w += __uint_as_float(rr.w);
          acc_out[i] = a;
        }
      }
      if (job.ticket != nullptr) {
        asm volatile("bar.sync 2, 64;" ::: "memory");      // this CTA's share is written
        if (aux_tid == 0 && last_cta_arrives(job.ticket)) {
          for (int i = 0; i < job.sig_n; ++i) release_store_sys(job.sig_ptrs[i], job.sig_value);
          if (job.done_flag != nullptr)
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(job.done_flag), "r"(job.done_value) : "memory");
        }
      }
    }
    if (tracer) {
      p.aux_trace[1] = waited_until;
      p.aux_trace[2] = globaltimer_ns();
    }
  }

  // ===================================== teardown =====================================
  if constexpr (kCS > 1) {
    cluster_sync_all();   // peers may still multicast into this CTA's smem / arrive on its barriers
  } else {
    __syncthreads();
  }
  // every warp of this CTA is past its last global write (barrier above): the last CTA of the launch tells the peers
  if (threadIdx.x == 0 && p.aux_trace != nullptr) atomicMin(p.aux_trace + 8, globaltimer_ns());   // first CTA to finish
  if (threadIdx.x == 0 && p.end_ticket != nullptr) {
    if (last_cta_arrives(p.end_ticket)) {
      for (int i = 0; i < p.end_sig_n; ++i) release_store_sys(p.end_sig_ptrs[i], p.end_sig_value);
      if (p.aux_trace != nullptr) p.aux_trace[3] = globaltimer_ns();
    }
  }
}

// -------------------------------------------------------------------------------------------------
// small helper kernels
// -------------------------------------------------------------------------------------------------
__global__ void reduce_slots_kernel(void* __restrict__ out, int out_bf16, const float* const* __restrict__ slots,
                                    int nslots, size_t n4) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 acc = reinterpret_cast<const float4*>(slots[0])[i];
    for (int s = 1; s < nslots; ++s) {
      const float4 v = reinterpret_cast<const float4*>(slots[s])[i];
      acc.x += v.x;
      acc.y += v.y;
      acc.z += v.z;
      acc.w += v.w;
    }
    if (out_bf16) {
      reinterpret_cast<uint2*>(out)[i] = make_uint2(pack_16x2<false>(acc.x, acc.y), pack_16x2<false>(acc.z, acc.w));
    } else {
      reinterpret_cast<float4*>(out)[i] = acc;
    }
  }
}

// dst = src * (*g): the whole backward() of the module when the fused step already produced the gradients for an
// upstream gradient of 1. 16-byte vectors when both buffers are 16-byte aligned, element-wise head / tail otherwise.
__device__ __forceinline__ uint4 scale_vec(uint4 v, int is_bf16, float s) {
  if (is_bf16) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t r[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      r[q] = pack_16x2<false>(__uint_as_float(w[q] << 16) * s, __uint_as_float(w[q] & 0xffff0000u) * s);
    return make_uint4(r[0], r[1], r[2], r[3]);
  }
  return make_uint4(__float_as_uint(__uint_as_float(v.x) * s), __float_as_uint(__uint_as_float(v.y) * s),
                    __float_as_uint(__uint_as_float(v.z) * s), __float_as_uint(__uint_as_float(v.w) * s));
}

__global__ void scale_kernel(const void* __restrict__ src, void* __restrict__ dst, int is_bf16,
                             const float* __restrict__ g, size_t nbytes, int aligned) {
  const float s = *g;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nvec = aligned ? nbytes / 16 : 0;
  for (size_t i = tid; i < nvec; i += stride)
    reinterpret_cast<uint4*>(dst)[i] = scale_vec(reinterpret_cast<const uint4*>(src)[i], is_bf16, s);
  // elements the vector loop did not cover (everything for unaligned buffers, < 16 bytes otherwise)
  const size_t esz = is_bf16 ? 2 : 4;
  const size_t first = nvec * 16 / esz, nel = nbytes / esz;
  for (size_t i = first + tid; i < nel; i += stride) {
    if (is_bf16) {
      const __nv_bfloat16 x = reinterpret_cast<const __nv_bfloat16*>(src)[i];
      reinterpret_cast<__nv_bfloat16*>(dst)[i] = __float2bfloat16_rn(__bfloat162float(x) * s);
    } else {
      reinterpret_cast<float*>(dst)[i] = reinterpret_cast<const float*>(src)[i] * s;
    }
  }
}

__global__ void signal_flags_kernel(unsigned int* const* flag_ptrs, int n, unsigned int value) {
  // everything this stream wrote before the signal must be visible to the peers that observe the flag
  __threadfence_system();
  const int i = threadIdx.x;
  if (i < n) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag_ptrs[i]), "r"(value) : "memory");
  }
}

__global__ void wait_flags_kernel(const volatile unsigned int* flags, int n, unsigned int value,
                                  unsigned long long timeout_ns, DebugRecord* dbg) {
  const int i = threadIdx.x;
  if (i < n) {
    uint64_t t0 = 0;
    uint32_t spins = 0;
    while (true) {
      unsigned int v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + i) : "memory");
      if (v >= value) break;
      if ((++spins & 0xffu) == 0) {
        const uint64_t now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        if (now - t0 > timeout_ns) {
          if (dbg != nullptr) {
            dbg->block = i;
            dbg->aux0 = v;
            dbg->aux1 = value;
            dbg->code = 6;
            __threadfence_system();
          }
          __trap();
        }
      }
    }
  }
}

// Mean over the ranks of the two scalar gradients (SURVEY.md §8f-2): what wrapping the module in DDP (README.md:20) or
// the toy average_gradients (test_distributed_sigmoid_loss.py:79-83) does with an all_reduce, here as one warp that
// publishes (dt', dbias) in a peer-visible mailbox, signals every rank, waits for every rank and adds the W mailboxes
// in rank order — the same order on every rank, so all ranks end up with bit-identical parameter gradients.
__global__ void allreduce_scalars_kernel(const float* __restrict__ saved, const float* __restrict__ g,
                                         float* mailbox_local, const float* const* __restrict__ mailboxes,
                                         unsigned int* const* __restrict__ signal_ptrs,
                                         const volatile unsigned int* flags_local, int world, unsigned int value,
                                         float* dt_prime, float* dbias, int dtp_f64, unsigned long long timeout_ns,
                                         DebugRecord* dbg) {
  __shared__ float sh[2][32];
  const int i = threadIdx.x;
  const float s = (g != nullptr) ? *g : 1.0f;
  if (i == 0) {
    asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mailbox_local), "f"(saved[0] * s) : "memory");
    asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mailbox_local + 1), "f"(saved[1] * s) : "memory");
    __threadfence_system();
  }
  __syncwarp();
  if (i < world) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(signal_ptrs[i]), "r"(value) : "memory");
    uint64_t t0 = 0;
    uint32_t spins = 0;
    while (true) {
      unsigned int v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags_local + i) : "memory");
      if (v >= value) break;
      if ((++spins & 0xffu) == 0) {
        const uint64_t now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        if (now - t0 > timeout_ns) {
          if (dbg != nullptr) {
            dbg->block = i;
            dbg->aux0 = v;
            dbg->aux1 = value;
            dbg->code = 9;
            __threadfence_system();
          }
          __trap();
        }
      }
    }
    float a, b;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(a) : "l"(mailboxes[i]) : "memory");
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(b) : "l"(mailboxes[i] + 1) : "memory");
    sh[0][i] = a;
    sh[1][i] = b;
  }
  __syncwarp();
  if (i == 0) {
    float a = 0.0f, b = 0.0f;
    for (int p = 0; p < world; ++p) {
      a += sh[0][p];
      b += sh[1][p];
    }
    const float inv_w = 1.0f / static_cast<float>(world);
    if (dt_prime) {
      if (dtp_f64)
        *reinterpret_cast<double*>(dt_prime) = static_cast<double>(a * inv_w);
      else
        *dt_prime = a * inv_w;
    }
    if (dbias) *dbias = b * inv_w;
  }
}

// Finalisation of a metrics step, one block. W > 1 follows allreduce_scalars_kernel: publish (flag kind 5 = step) that my
// column partials are complete, wait for every rank's, then max-combine the W partials of my chunk with relaxed
// system-scope loads. It never triggers griddepcontrol.launch_dependents: the next step's first loss kernel (launched
// with programmatic serialization) cannot touch global memory before this kernel has ended (DESIGN.md, "In-batch
// retrieval metrics").
constexpr int kMetricsThreads = 1024;

// owner rank of global index g under the prefix sums `off` (images: a.off, texts: a.toff)
__device__ __forceinline__ int metrics_owner(const MetricsArgs& a, const int* off, int g) {
  int o = 0;
  while (o + 1 < a.world && g >= off[o + 1]) ++o;
  return o;
}

// sample id of the l-th sample of rank o (its image and its paired text share it); under extra_ids, l >= B_o is the id
// of its text l
__device__ __forceinline__ int64_t metrics_id(const MetricsArgs& a, int o, int l) {
  return (o == a.rank) ? a.ids_own[l] : a.ids_all[static_cast<size_t>(o) * a.ids_stride + l];
}

// Is global text j a hit for my image i? The positional pair, or with ids a text with the same id. Only the paired texts
// carry ids unless extra_ids: a hard negative (local text index >= its rank's batch) then never is a hit, so one that
// outranks the caption counts as a miss. Under extra_ids every text of rank o (l < T_o) carries one.
__device__ __forceinline__ bool metrics_i2t_hit(const MetricsArgs& a, int i, int j) {
  if (a.ids_own == nullptr) return j == a.toff[a.rank] + i;
  const int o = metrics_owner(a, a.toff, j);
  const int l = j - a.toff[o];
  const int with_ids = a.extra_ids ? a.toff[o + 1] - a.toff[o] : a.bs[o];
  return l < with_ids && metrics_id(a, o, l) == a.row_ids[i];
}

// Is global image g a hit for my text i (a paired one, or any under extra_ids)? An extra image (local index >= its
// rank's batch) carries an id only under extra_image_ids: its owner's row ids, or the copy that owner published.
__device__ __forceinline__ bool metrics_t2i_hit(const MetricsArgs& a, int i, int g) {
  if (a.ids_own == nullptr) return g == a.off[a.rank] + i;
  const int o = metrics_owner(a, a.off, g);
  const int l = g - a.off[o];
  if (l < a.bs[o]) return metrics_id(a, o, l) == a.ids_own[i];
  if (!a.extra_image_ids) return false;
  int64_t id;
  if (o == a.rank) {
    id = a.row_ids[l];
  } else {
    asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(id) : "l"(a.xids_peers[o] + (l - a.bs[o])) : "memory");
  }
  return id == a.ids_own[i];
}

// ---- label sets (SIGLIP_OPT_LABEL_SETS): the hit rule of the kLabels finalisations ----
// Do the set x (kMaxLabels entries, -1 past m) and the m labels at y share a label >= 0? kPeer: y lies in a peer's
// memory and is read with relaxed system-scope loads.
template <bool kPeer = false>
__device__ __forceinline__ bool label_sets_meet(const int64_t (&x)[kMaxLabels], const int64_t* y, int m) {
  bool hit = false;
  for (int k = 0; k < m; ++k) {
    int64_t v;
    if constexpr (kPeer)
      asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(y + k) : "memory");
    else
      v = y[k];
    if (v < 0) continue;
#pragma unroll
    for (int q = 0; q < kMaxLabels; ++q) hit |= v == x[q];
  }
  return hit;
}
__device__ __forceinline__ void label_set_load(int64_t (&x)[kMaxLabels], const int64_t* s, int m) {
#pragma unroll
  for (int k = 0; k < kMaxLabels; ++k) x[k] = k < m ? s[k] : -1;
}
// the sets of text l of rank o as this rank holds them: its own, or the gathered copy
__device__ __forceinline__ const int64_t* label_text_set(const MetricsArgs& a, const LabelSetArgs& l, int o, int t) {
  return ((o == a.rank) ? l.text_own : l.text_all + static_cast<size_t>(o) * l.slot) + static_cast<size_t>(t) * l.m;
}
// Is global text j a hit for my image i? The positional pair, or a text whose set meets the image's.
__device__ __forceinline__ bool labels_i2t_hit(const MetricsArgs& a, const LabelSetArgs& l, int i, int j) {
  const int o = metrics_owner(a, a.toff, j);
  const int t = j - a.toff[o];
  if (o == a.rank && t == i && i < a.B) return true;
  int64_t x[kMaxLabels];
  label_set_load(x, l.row_sets + static_cast<size_t>(i) * l.m, l.m);
  return label_sets_meet(x, label_text_set(a, l, o, t), l.m);
}
// Is global image g a hit for my text i? The positional pair, or an image whose set meets the text's: a paired image
// shares its paired text's set (the gathered copy), an extra image of a peer is read from the sets that peer published.
__device__ __forceinline__ bool labels_t2i_hit(const MetricsArgs& a, const LabelSetArgs& l, int i, int g) {
  const int o = metrics_owner(a, a.off, g);
  const int r = g - a.off[o];
  if (o == a.rank && r == i && i < a.B) return true;
  int64_t x[kMaxLabels];
  label_set_load(x, l.text_own + static_cast<size_t>(i) * l.m, l.m);
  if (o == a.rank) return label_sets_meet(x, l.row_sets + static_cast<size_t>(r) * l.m, l.m);
  if (r < a.bs[o]) return label_sets_meet(x, label_text_set(a, l, o, r), l.m);
  return label_sets_meet<true>(x, l.xsets_peers[o] + static_cast<size_t>(r - a.bs[o]) * l.m, l.m);
}
template <bool kLabels>
__device__ __forceinline__ bool finalize_i2t_hit(const MetricsArgs& a, const LabelSetArgs& l, int i, int j) {
  if constexpr (kLabels)
    return labels_i2t_hit(a, l, i, j);
  else
    return metrics_i2t_hit(a, i, j);
}
template <bool kLabels>
__device__ __forceinline__ bool finalize_t2i_hit(const MetricsArgs& a, const LabelSetArgs& l, int i, int g) {
  if constexpr (kLabels)
    return labels_t2i_hit(a, l, i, g);
  else
    return metrics_t2i_hit(a, i, g);
}

__device__ __forceinline__ int key_index(unsigned long long k) {
  return k == 0ull ? -1 : static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(k));
}

// kLabels: the hit rule of a label-set step (LabelSetArgs); the kernel without it is metrics_finalize_kernel below
template <bool kLabels>
__device__ __forceinline__ void metrics_finalize(const MetricsArgs& a, const LabelSetArgs& l) {
  __shared__ unsigned int hits[2];
  const int tid = threadIdx.x;
  if (tid < 2) hits[tid] = 0u;
  if (a.world > 1) {
    if (tid < a.world) {
      __threadfence_system();   // my partials (written by the step's loss kernels) before the flag
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.sig_ptrs[tid]), "r"(a.value) : "memory");
      uint64_t t0 = 0;
      uint32_t spins = 0;
      while (true) {
        unsigned int v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a.flags_local + tid) : "memory");
        if (v >= a.value) break;
        if ((++spins & 0xffu) == 0) {
          const uint64_t now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          if (now - t0 > a.timeout_ns) {
            if (a.dbg != nullptr) {
              a.dbg->block = tid;
              a.dbg->aux0 = v;
              a.dbg->aux1 = a.value;
              a.dbg->code = 10;
              __threadfence_system();
            }
            __trap();
          }
        }
      }
      __threadfence();   // order the other threads' peer reads after the observed flags
    }
  }
  __syncthreads();
  unsigned int h_i2t = 0, h_t2i = 0;
  // column partials are read for the paired texts (i < B), and under extra_ids or label sets for every text of this
  // rank (i < T); otherwise the extras' column keys are computed but never read
  const int nt = (kLabels || a.extra_ids) ? a.T : a.B;
  // images ranked by i2t: the paired ones, and under extra_image_ids or label sets every image of this rank (row keys
  // of the extras are computed but never read otherwise)
  const int ni = (kLabels || a.extra_image_ids) ? a.R : a.B;
  const int n = ni > nt ? ni : nt;
  for (int i = tid; i < n; i += kMetricsThreads) {
    if (i < ni) {
      const int j = key_index(a.row_keys[i]);   // best text of my image i, over all texts including the extras
      if (a.i2t) a.i2t[i] = j;
      if (j >= 0) h_i2t += finalize_i2t_hit<kLabels>(a, l, i, j);
    }
    if (i >= nt) continue;
    unsigned long long k = a.col_own[i];
    if (a.world > 1) {
      for (int q = 0; q < a.world; ++q) {
        if (q == a.rank) continue;
        unsigned long long v;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(a.col_peers[q] + i) : "memory");
        k = max_u64(k, v);
      }
    }
    const int g = key_index(k);               // best image of my text i
    if (a.t2i) a.t2i[i] = g;
    if (g >= 0) h_t2i += finalize_t2i_hit<kLabels>(a, l, i, g);
  }
  // integer counts: the sum does not depend on the order
  for (int o = 16; o > 0; o >>= 1) {
    h_i2t += __shfl_xor_sync(0xffffffffu, h_i2t, o);
    h_t2i += __shfl_xor_sync(0xffffffffu, h_t2i, o);
  }
  if ((tid & 31) == 0) {
    atomicAdd(&hits[0], h_i2t);
    atomicAdd(&hits[1], h_t2i);
  }
  __syncthreads();
  if (tid < 2) a.top1[tid] = static_cast<float>(hits[tid]) / static_cast<float>(tid == 0 ? ni : nt);
}

__global__ void __launch_bounds__(kMetricsThreads) metrics_finalize_kernel(const MetricsArgs a) {
  metrics_finalize<false>(a, LabelSetArgs{});
}
__global__ void __launch_bounds__(kMetricsThreads) metrics_finalize_labels_kernel(const MetricsArgs a,
                                                                                  const LabelSetArgs l) {
  metrics_finalize<true>(a, l);
}

// Finalisation of the per-sample losses (SampleLossArgs). Like metrics_finalize_kernel it never triggers
// griddepcontrol.launch_dependents, and at W > 1 it reads the peers' partials of the step only after their flag kind 5
// of the step: the same words at the same points of the step as the metric keys (DESIGN.md, "Per-sample losses").
constexpr int kSampleLossThreads = 1024;

__device__ __forceinline__ float sample_loss_decode(unsigned long long sum, unsigned long long poison) {
  if (poison & 2ull) return __int_as_float(0x7fffffff);
  if (poison & 1ull) return INFINITY;
  return static_cast<float>(static_cast<double>(sum) * (1.0 / kSampleLossScale));
}

__global__ void __launch_bounds__(kSampleLossThreads) sample_loss_finalize_kernel(const SampleLossArgs a) {
  const int tid = threadIdx.x;
  if (a.world > 1) {
    if (tid < a.world) {
      if (a.signal) {
        __threadfence_system();   // my partials (written by the step's loss kernels) before the flag
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.sig_ptrs[tid]), "r"(a.value) : "memory");
      }
      uint64_t t0 = 0;
      uint32_t spins = 0;
      while (true) {
        unsigned int v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a.flags_local + tid) : "memory");
        if (v >= a.value) break;
        if ((++spins & 0xffu) == 0) {
          const uint64_t now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          if (now - t0 > a.timeout_ns) {
            if (a.dbg != nullptr) {
              a.dbg->block = tid;
              a.dbg->aux0 = v;
              a.dbg->aux1 = a.value;
              a.dbg->code = 10;
              __threadfence_system();
            }
            __trap();
          }
        }
      }
      __threadfence();   // order the other threads' peer reads after the observed flags
    }
    __syncthreads();
  }
  for (int i = tid; i < a.R; i += kSampleLossThreads) a.image_loss[i] = sample_loss_decode(a.rows[i], a.rows[i + a.poison]);
  for (int i = tid; i < a.T; i += kSampleLossThreads) {
    unsigned long long sum = a.col_own[i], poison = a.col_own[i + a.poison];
    if (a.world > 1) {
      for (int q = 0; q < a.world; ++q) {   // integer sums: the rank order is only for definiteness
        if (q == a.rank) continue;
        unsigned long long v, b;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(a.col_peers[q] + i) : "memory");
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(b) : "l"(a.col_peers[q] + i + a.poison) : "memory");
        sum += v;
        poison |= b;
      }
    }
    a.text_loss[i] = sample_loss_decode(sum, poison);
  }
}

// Finalisation of a top-K step (TopKArgs). Like metrics_finalize_kernel it never triggers
// griddepcontrol.launch_dependents, and at W > 1 it reads the peers' lists of the step only after their flag kind 5 of
// the step: the same protocol as the metric keys (DESIGN.md, "Top-K retrieval").
constexpr int kTopKThreads = 1024;

// kLabels: the hit rule of a label-set step (LabelSetArgs); the kernel without it is topk_finalize_kernel below
template <bool kLabels>
__device__ __forceinline__ void topk_finalize(const TopKArgs& t, const LabelSetArgs& l) {
  const MetricsArgs& a = t.m;
  // first[side][s]: samples whose first hit is at rank s (s = K: no hit among the K)
  __shared__ unsigned int first[2][kTopKMax + 1];
  const int tid = threadIdx.x;
  if (tid < 2 * (kTopKMax + 1)) first[tid / (kTopKMax + 1)][tid % (kTopKMax + 1)] = 0u;
  if (a.world > 1) {
    if (tid < a.world) {
      if (t.signal) {
        __threadfence_system();   // my lists (written by the step's loss kernels) before the flag
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a.sig_ptrs[tid]), "r"(a.value) : "memory");
      }
      uint64_t t0 = 0;
      uint32_t spins = 0;
      while (true) {
        unsigned int v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a.flags_local + tid) : "memory");
        if (v >= a.value) break;
        if ((++spins & 0xffu) == 0) {
          const uint64_t now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          if (now - t0 > a.timeout_ns) {
            if (a.dbg != nullptr) {
              a.dbg->block = tid;
              a.dbg->aux0 = v;
              a.dbg->aux1 = a.value;
              a.dbg->code = 10;
              __threadfence_system();
            }
            __trap();
          }
        }
      }
      __threadfence();   // order the other threads' peer reads after the observed flags
    }
  }
  __syncthreads();
  const int K = t.k;
  // the images and texts ranked, as in metrics_finalize
  const int nt = (kLabels || a.extra_ids) ? a.T : a.B;
  const int ni = (kLabels || a.extra_image_ids) ? a.R : a.B;
  const int n = ni > nt ? ni : nt;
  unsigned int cnt[2][kTopKMax + 1] = {};   // per thread, by first-hit rank (K: none)
  for (int i = tid; i < n; i += kTopKThreads) {
    unsigned long long key[kTopKMax];
    if (i < ni) {
#pragma unroll
      for (int s = 0; s < kTopKMax; ++s) key[s] = (s < K) ? t.rows[static_cast<size_t>(i) * kTopKMax + s] : 0ull;
      int f = K;
#pragma unroll
      for (int s = 0; s < kTopKMax; ++s) {
        if (s < K) {
          const int j = key_index(key[s]);
          if (t.i2t) t.i2t[static_cast<size_t>(i) * K + s] = j;
          if (f == K && j >= 0 && finalize_i2t_hit<kLabels>(a, l, i, j)) f = s;
        }
      }
#pragma unroll
      for (int s = 0; s <= kTopKMax; ++s) cnt[0][s] += (f == s);
    }
    if (i >= nt) continue;
    if (a.world == 1) {
#pragma unroll
      for (int s = 0; s < kTopKMax; ++s) key[s] = (s < K) ? t.col_own[static_cast<size_t>(i) * kTopKMax + s] : 0ull;
    } else {
      // K-way merge of the W sorted lists (keys of different ranks are distinct: each covers that rank's images): the
      // head of every list is kept, and only the list whose head was taken is read again
      int head[kMetricsMaxWorld] = {};
      unsigned long long hv[kMetricsMaxWorld];
      auto load = [&](int q) -> unsigned long long {
        if (head[q] >= K) return 0ull;
        const size_t o = static_cast<size_t>(i) * kTopKMax + head[q];
        if (q == a.rank) return t.col_own[o];
        unsigned long long v;
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(t.col_peers[q] + o) : "memory");
        return v;
      };
      for (int q = 0; q < a.world; ++q) hv[q] = load(q);
#pragma unroll
      for (int s = 0; s < kTopKMax; ++s) {
        unsigned long long best = 0ull;
        int bq = -1;
        if (s < K) {
          for (int q = 0; q < a.world; ++q) {
            if (hv[q] > best) {
              best = hv[q];
              bq = q;
            }
          }
          if (bq >= 0) {
            ++head[bq];
            hv[bq] = load(bq);
          }
        }
        key[s] = best;
      }
    }
    int f = K;
#pragma unroll
    for (int s = 0; s < kTopKMax; ++s) {
      if (s < K) {
        const int g = key_index(key[s]);
        if (t.t2i) t.t2i[static_cast<size_t>(i) * K + s] = g;
        if (f == K && g >= 0 && finalize_t2i_hit<kLabels>(a, l, i, g)) f = s;
      }
    }
#pragma unroll
    for (int s = 0; s <= kTopKMax; ++s) cnt[1][s] += (f == s);
  }
  // integer counts: the sum does not depend on the order
#pragma unroll
  for (int d = 0; d < 2; ++d) {
#pragma unroll
    for (int s = 0; s <= kTopKMax; ++s) {
      unsigned int v = cnt[d][s];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((tid & 31) == 0 && v != 0u) atomicAdd(&first[d][s], v);
    }
  }
  __syncthreads();
  // recall@k = (samples with their first hit at a rank < k) / samples: integer counts, as the top-1 rate
  if (tid < 2) {
    unsigned int hits = 0u;
    for (int s = 0; s < K; ++s) {
      hits += first[tid][s];
      t.recall[tid * K + s] = static_cast<float>(hits) / static_cast<float>(tid == 0 ? ni : nt);
    }
  }
}

__global__ void __launch_bounds__(kTopKThreads) topk_finalize_kernel(const TopKArgs t) {
  topk_finalize<false>(t, LabelSetArgs{});
}
__global__ void __launch_bounds__(kTopKThreads) topk_finalize_labels_kernel(const TopKArgs t, const LabelSetArgs l) {
  topk_finalize<true>(t, l);
}

// -------------------------------------------------------------------------------------------------
// L2 normalisation fused around the loss (SURVEY.md §8f-1: the step the reference's callers run right before it,
// test_distributed_sigmoid_loss.py:99-101). One warp per row; HBM-bound: coalesced 16-byte accesses, fp32 math.
// -------------------------------------------------------------------------------------------------
template <bool kInBf16>
__device__ __forceinline__ void load8(const void* base, size_t idx8, float (&v)[8]) {
  if constexpr (kInBf16) {
    const uint4 w = reinterpret_cast<const uint4*>(base)[idx8];
    const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      v[2 * q] = __uint_as_float(u[q] << 16);
      v[2 * q + 1] = __uint_as_float(u[q] & 0xffff0000u);
    }
  } else {
    const float4 a = reinterpret_cast<const float4*>(base)[2 * idx8];
    const float4 b = reinterpret_cast<const float4*>(base)[2 * idx8 + 1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
}

template <bool kOutBf16>
__device__ __forceinline__ void store8(void* base, size_t idx8, const float (&v)[8]) {
  if constexpr (kOutBf16) {
    reinterpret_cast<uint4*>(base)[idx8] = make_uint4(pack_16x2<false>(v[0], v[1]), pack_16x2<false>(v[2], v[3]),
                                                      pack_16x2<false>(v[4], v[5]), pack_16x2<false>(v[6], v[7]));
  } else {
    reinterpret_cast<float4*>(base)[2 * idx8] = make_float4(v[0], v[1], v[2], v[3]);
    reinterpret_cast<float4*>(base)[2 * idx8 + 1] = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// fp16(v * scale), finite values clamped to the fp16 range, NaN and +-inf kept: the operand format of the fp32-input path
__device__ __forceinline__ void store8_f16(void* base, size_t idx8, const float (&v)[8], float scale) {
  uint32_t o[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) o[q] = pack_f16x2_scaled(v[2 * q], v[2 * q + 1], scale);
  reinterpret_cast<uint4*>(base)[idx8] = make_uint4(o[0], o[1], o[2], o[3]);
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// xhat[r, :] = bf16(x[r, :] / max(||x[r, :]||, eps)),  inv_norm[r] = 1 / max(||x||, eps)      (F.normalize, eps 1e-12)
// f16_scale > 0: xhat is written as fp16(xhat * f16_scale) instead of bf16 (fp32-input path)
template <bool kInBf16>
__global__ void normalize_fwd_kernel(const void* __restrict__ x, __nv_bfloat16* __restrict__ xhat,
                                     float* __restrict__ inv_norm, int rows, int d8, float f16_scale) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < rows; r += gridDim.x * warps_per_block) {
    const size_t row8 = static_cast<size_t>(r) * d8;
    float ss = 0.f;
    for (int c = lane; c < d8; c += 32) {
      float v[8];
      load8<kInBf16>(x, row8 + c, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) ss = fmaf(v[e], v[e], ss);
    }
    ss = warp_sum_f(ss);
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
    if (lane == 0) inv_norm[r] = inv;
    for (int c = lane; c < d8; c += 32) {
      float v[8];
      load8<kInBf16>(x, row8 + c, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] *= inv;
      if (f16_scale > 0.f)
        store8_f16(xhat, row8 + c, v, f16_scale);
      else
        store8<true>(xhat, row8 + c, v);
    }
  }
}

// dst = bf16(src) or fp16(src * f16_scale): the module's cast of fp32 embeddings to the operand format
__global__ void convert_f32_kernel(const float* __restrict__ src, void* __restrict__ dst, size_t n8, float f16_scale) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
    float v[8];
    load8<false>(src, i, v);
    if (f16_scale > 0.f)
      store8_f16(dst, i, v, f16_scale);
    else
      store8<true>(dst, i, v);
  }
}

// dx = inv * (dxhat - xhat * <xhat, dxhat>) with xhat = x * inv recomputed in fp32 from the raw input
template <bool kInBf16, bool kGradBf16>
__global__ void normalize_bwd_kernel(const void* __restrict__ x, const float* __restrict__ inv_norm,
                                     const void* __restrict__ dxhat, void* __restrict__ dx, int rows, int d8) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int r = blockIdx.x * warps_per_block + (threadIdx.x >> 5); r < rows; r += gridDim.x * warps_per_block) {
    const size_t row8 = static_cast<size_t>(r) * d8;
    const float inv = inv_norm[r];
    float dot = 0.f;
    for (int c = lane; c < d8; c += 32) {
      float v[8], g[8];
      load8<kInBf16>(x, row8 + c, v);
      load8<kGradBf16>(dxhat, row8 + c, g);
#pragma unroll
      for (int e = 0; e < 8; ++e) dot = fmaf(v[e] * inv, g[e], dot);
    }
    dot = warp_sum_f(dot);
    for (int c = lane; c < d8; c += 32) {
      float v[8], g[8], o[8];
      load8<kInBf16>(x, row8 + c, v);
      load8<kGradBf16>(dxhat, row8 + c, g);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = inv * (g[e] - v[e] * inv * dot);
      store8<kInBf16>(dx, row8 + c, o);
    }
  }
}

// kIds / kMetrics / kWeights select the sample-id / retrieval-metrics / sample-weight instantiations of the loss kernel
// (ignored for the out kernel); kTileNT the column-tile width
template <int kMode, int kStages, int kCS, bool kF8 = false, bool kIds = false, bool kMetrics = false,
          bool kWeights = false, int kTileNT = kTileN>
int launch_impl(const CUtensorMap* tmA0, const CUtensorMap* tmB0, const CUtensorMap* tmA1, const CUtensorMap* tmB1,
                const CUtensorMap* tmG, const KernelParams& p, int num_sms, cudaStream_t stream) {
  using C = Cfg<kMode, kStages, kTileNT>;
  auto kern = siglip_gemm_kernel<kMode, kStages, kCS, kF8, kIds && kMode == kModeLoss, kMetrics && kMode == kModeLoss,
                                 kWeights && kMode == kModeLoss, kTileNT>;   // kModeDistill: runtime options
  static bool attr_set = false;
  cudaError_t e = cudaSuccess;
  if (!attr_set) {
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes);
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set = true;
  }
  KernelParams pl = p;
  int total_tiles = 0;
  for (int i = 0; i < pl.nprob; ++i) {
    Problem& pr = pl.prob[i];
    pr.tiles_m = (pr.M + kBlockM * kCS - 1) / (kBlockM * kCS);
    pr.tiles_n = (pr.N + kTileNT - 1) / kTileNT;
    total_tiles += pr.tiles_m * pr.tiles_n;
  }
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = C::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  // A persistent kernel must have every cluster co-resident: clusters of 4 do not tile every GPC, so ask the runtime
  // how many fit (once per instantiation) instead of assuming num_sms / cluster size.
  static int max_clusters = -1;
  if (max_clusters < 0) {
    cfg.gridDim = dim3((num_sms / kCS) * kCS);
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = num_sms / kCS;
    }
    max_clusters = n;
    if (getenv("SIGLIP_DEBUG_WAITSTATS")) printf("[launch] cluster size %d: %d co-resident clusters\n", kCS, n);
  }
  int clusters = max_clusters < num_sms / kCS ? max_clusters : num_sms / kCS;
  pl.sk_parts = 0;
  if (kMode == kModeOut && kTileNT == kTileN && p.sk_request != 0 && p.sk_ws != nullptr && clusters > 1) {
    // Split-K of the ragged last wave: `rem` tiles left after the full waves would occupy rem of `clusters` units for
    // a whole tile time. Cut each of them into S = floor(clusters / rem) K-slices (S * rem <= clusters work items, one
    // per unit): the last wave then lasts ~1/S of a tile. Not worth it when the last wave is more than half full
    // (S would be 1) or the slices get shorter than a handful of k-blocks.
    const int rem = total_tiles % clusters;
    const int min_k = pl.prob[0].K < pl.prob[pl.nprob > 1 ? 1 : 0].K ? pl.prob[0].K : pl.prob[pl.nprob > 1 ? 1 : 0].K;
    const int num_kb = (min_k + kBlockK - 1) / kBlockK;
    if (rem > 0) {
      int S = clusters / rem;
      if (p.sk_request > 1 && S > p.sk_request) S = p.sk_request;
      if (p.sk_request < 0 && S > 4) S = 4;
      while (S > 1 && num_kb / S < 8) --S;
      const size_t need = static_cast<size_t>(rem) * (S - 1) * kCS * kBlockM * kTileN * sizeof(float);
      if (S >= 2 && rem <= p.sk_max_tiles && need <= p.sk_ws_bytes) {
        pl.sk_parts = S;
        pl.sk_tiles = rem;
        pl.sk_first = total_tiles - rem;
        total_tiles = pl.sk_first + rem * S;
      }
    }
  }
  // a loss launch keeps the grid of the largest chunk of its forward (KernelParams::grid_n): CTA i owns partial slot i
  // in every chunk, and the CTAs without a tile only carry their slot forward
  int grid_tiles = total_tiles;
  if (kMode != kModeOut && pl.grid_n > pl.prob[0].N)
    grid_tiles = pl.prob[0].tiles_m * ((pl.grid_n + kTileN - 1) / kTileN);
  if (clusters > grid_tiles) clusters = grid_tiles;
  if (clusters < 1) clusters = 1;
  cfg.gridDim = dim3(clusters * kCS);
  cfg.numAttrs = pl.pdl ? 2 : 1;
  e = cudaLaunchKernelEx(&cfg, kern, *tmA0, *tmB0, *tmA1, *tmB1, *tmG, pl);
  return static_cast<int>(e);
}

}  // namespace

int query_max_active_clusters(int cluster) {
  int n = -1, dev = 0, num_sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return n;
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cfg.blockDim = dim3(kNumThreads);
  cfg.gridDim = dim3((num_sms / cluster) * cluster);
  cfg.dynamicSmemBytes = Cfg<kModeOut, 6>::kSmemBytes;
  auto query = [&](auto kern) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cfg.dynamicSmemBytes);
    cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
  };
  if (cluster == 4)
    query(siglip_gemm_kernel<kModeOut, 6, 4>);
  else if (cluster == 2)
    query(siglip_gemm_kernel<kModeOut, 6, 2>);
  else
    query(siglip_gemm_kernel<kModeOut, 6, 1>);
  return n;
}

int default_stages(int /*mode*/) { return 6; }

size_t gemm_smem_bytes(int mode) {
  return mode == kModeLoss ? static_cast<size_t>(Cfg<kModeLoss, 6>::kSmemBytes)
                           : static_cast<size_t>(Cfg<kModeOut, 6>::kSmemBytes);
}

// the out kernel never has ids, metric keys or weights, so only the loss kernel takes the seven extra instantiations
#define SIGLIP_LAUNCH(MODE, ST, CS)                                                                          \
  do {                                                                                                       \
    const bool ids__ = p.row_ids != nullptr, met__ = p.row_keys != nullptr;                                  \
    if (MODE == kModeLoss && p.row_w != nullptr) {                                                           \
      if (ids__ && met__) return launch_impl<MODE, ST, CS, false, true, true, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream); \
      if (met__) return launch_impl<MODE, ST, CS, false, false, true, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);        \
      if (ids__) return launch_impl<MODE, ST, CS, false, true, false, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);        \
      return launch_impl<MODE, ST, CS, false, false, false, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);                  \
    }                                                                                                        \
    if (ids__ && met__) return launch_impl<MODE, ST, CS, false, true, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream); \
    if (met__) return launch_impl<MODE, ST, CS, false, false, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);        \
    if (ids__) return launch_impl<MODE, ST, CS, false, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);               \
    return launch_impl<MODE, ST, CS>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);                                      \
  } while (0)

#define SIGLIP_LAUNCH_STAGES(MODE, CS)   \
  do {                                   \
    if (stages == 4) SIGLIP_LAUNCH(MODE, 4, CS); \
    SIGLIP_LAUNCH(MODE, 6, CS);          \
  } while (0)

// the five tensor maps and the parameter block travel as kernel parameters: keep them inside the classic 4 KiB limit
static_assert(5 * sizeof(CUtensorMap) + sizeof(KernelParams) <= 4096, "kernel parameters exceed 4 KiB");

// Distillation with per-sample losses, top-K, groups or label sets: kModeDistillOpts at kDistillStages. Defined behind
// launch_gemm, so that its three kernels come after every other kernel in the module, whose code stays as it was.
static int launch_distill_opts(int cluster, const CUtensorMap* tmA0, const CUtensorMap* tmB0, const CUtensorMap* tmA1,
                               const CUtensorMap* tmB1, const CUtensorMap* tmG, const KernelParams& p, int num_sms,
                               cudaStream_t stream);

int launch_gemm(int cta_group, int mode, int stages, int mcast, int tile_n, const CUtensorMap* tmA0,
                const CUtensorMap* tmB0, const CUtensorMap* tmA1, const CUtensorMap* tmB1, const CUtensorMap* tmG,
                const KernelParams& p, int num_sms, cudaStream_t stream) {
  if (stages <= 0) stages = default_stages(mode);
  if (mode == kModeOut && p.prob[0].ab_f16 == 2) {   // 8-bit measurement path: K-major, no multicast, no split-K
    if (tile_n != kTileN) return static_cast<int>(cudaErrorInvalidValue);
    if (cluster_size(cta_group, mcast) == 2)
      return launch_impl<kModeOut, 6, 2, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    return launch_impl<kModeOut, 6, 1, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
  }
  if (tile_n == kWideTileN) {   // every stage request maps to the 4 stages that fit
    if (mode != kModeOut) return static_cast<int>(cudaErrorInvalidValue);
    switch (cluster_size(cta_group, mcast)) {
      case 4:
        return launch_impl<kModeOut, kWideStages, 4, false, false, false, false, kWideTileN>(tmA0, tmB0, tmA1, tmB1,
                                                                                            tmG, p, num_sms, stream);
      case 2:
        return launch_impl<kModeOut, kWideStages, 2, false, false, false, false, kWideTileN>(tmA0, tmB0, tmA1, tmB1,
                                                                                            tmG, p, num_sms, stream);
      default:
        return launch_impl<kModeOut, kWideStages, 1, false, false, false, false, kWideTileN>(tmA0, tmB0, tmA1, tmB1,
                                                                                            tmG, p, num_sms, stream);
    }
  }
  if (tile_n != kTileN) return static_cast<int>(cudaErrorInvalidValue);
  if (mode == kModeLoss && p.k_teacher > 0 &&
      (p.sl_rows != nullptr || p.tk_rows != nullptr || p.col_grp != nullptr || p.col_lab != nullptr))
    return launch_distill_opts(cluster_size(cta_group, mcast), tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
  if (mode == kModeLoss && p.k_teacher > 0) {   // distillation: kModeDistill, kDistillStages whatever `stages` asks
    switch (cluster_size(cta_group, mcast)) {
      case 4: return launch_impl<kModeDistill, kDistillStages, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      case 2: return launch_impl<kModeDistill, kDistillStages, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      default: return launch_impl<kModeDistill, kDistillStages, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    }
  }
  if (mode == kModeLoss && p.focal) {   // focal terms (with any option but distillation): kModeFocal
    const bool s4 = stages == 4;
    switch (cluster_size(cta_group, mcast)) {
      case 4:
        return s4 ? launch_impl<kModeFocal, 4, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeFocal, 6, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      case 2:
        return s4 ? launch_impl<kModeFocal, 4, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeFocal, 6, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      default:
        return s4 ? launch_impl<kModeFocal, 4, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeFocal, 6, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    }
  }
  if (mode == kModeLoss && p.col_lab != nullptr) {   // label sets (with any option but distillation): kModeLabels
    const bool s4 = stages == 4;
    switch (cluster_size(cta_group, mcast)) {
      case 4:
        return s4 ? launch_impl<kModeLabels, 4, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeLabels, 6, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      case 2:
        return s4 ? launch_impl<kModeLabels, 4, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeLabels, 6, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      default:
        return s4 ? launch_impl<kModeLabels, 4, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeLabels, 6, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    }
  }
  if (mode == kModeLoss && p.col_grp != nullptr) {   // excluded groups (with any other option): kModeGroups
    const bool s4 = stages == 4;
    switch (cluster_size(cta_group, mcast)) {
      case 4:
        return s4 ? launch_impl<kModeGroups, 4, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeGroups, 6, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      case 2:
        return s4 ? launch_impl<kModeGroups, 4, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeGroups, 6, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      default:
        return s4 ? launch_impl<kModeGroups, 4, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeGroups, 6, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    }
  }
  if (mode == kModeLoss && p.tk_rows != nullptr) {   // top-K (with or without per-sample losses): kModeTopK
    const bool s4 = stages == 4;
    switch (cluster_size(cta_group, mcast)) {
      case 4:
        return s4 ? launch_impl<kModeTopK, 4, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeTopK, 6, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      case 2:
        return s4 ? launch_impl<kModeTopK, 4, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeTopK, 6, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      default:
        return s4 ? launch_impl<kModeTopK, 4, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeTopK, 6, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    }
  }
  if (mode == kModeLoss && p.sl_rows != nullptr) {   // per-sample losses: kModeSampleLoss, 4 or 6 stages
    const bool s4 = stages == 4;
    switch (cluster_size(cta_group, mcast)) {
      case 4:
        return s4 ? launch_impl<kModeSampleLoss, 4, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeSampleLoss, 6, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      case 2:
        return s4 ? launch_impl<kModeSampleLoss, 4, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeSampleLoss, 6, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
      default:
        return s4 ? launch_impl<kModeSampleLoss, 4, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)
                  : launch_impl<kModeSampleLoss, 6, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    }
  }
  switch (cluster_size(cta_group, mcast)) {
    case 4:
      if (mode == kModeLoss) SIGLIP_LAUNCH_STAGES(kModeLoss, 4);
      SIGLIP_LAUNCH_STAGES(kModeOut, 4);
    case 2:
      if (mode == kModeLoss) SIGLIP_LAUNCH_STAGES(kModeLoss, 2);
      SIGLIP_LAUNCH_STAGES(kModeOut, 2);
    default:
      if (mode == kModeLoss) SIGLIP_LAUNCH_STAGES(kModeLoss, 1);
      SIGLIP_LAUNCH_STAGES(kModeOut, 1);
  }
}
#undef SIGLIP_LAUNCH_STAGES
#undef SIGLIP_LAUNCH

int launch_reduce_slots(void* out, int out_bf16, const float* const* slots_dev, int nslots, size_t n, int num_sms,
                        cudaStream_t stream) {
  reduce_slots_kernel<<<num_sms * 4, 256, 0, stream>>>(out, out_bf16, slots_dev, nslots, n / 4);
  return static_cast<int>(cudaGetLastError());
}

int launch_normalize_fwd(const void* x, int in_bf16, __nv_bfloat16* xhat, float* inv_norm, int rows, int D,
                         float f16_scale, int num_sms, cudaStream_t stream) {
  const int grid = num_sms * 8, block = 256;
  if (in_bf16)
    normalize_fwd_kernel<true><<<grid, block, 0, stream>>>(x, xhat, inv_norm, rows, D / 8, f16_scale);
  else
    normalize_fwd_kernel<false><<<grid, block, 0, stream>>>(x, xhat, inv_norm, rows, D / 8, f16_scale);
  return static_cast<int>(cudaGetLastError());
}

int launch_convert_f32(const float* src, void* dst, size_t n, float f16_scale, int num_sms, cudaStream_t stream) {
  convert_f32_kernel<<<num_sms * 4, 256, 0, stream>>>(src, dst, n / 8, f16_scale);
  return static_cast<int>(cudaGetLastError());
}

int launch_normalize_bwd(const void* x, int in_bf16, const float* inv_norm, const void* dxhat, int grad_bf16, void* dx,
                         int rows, int D, int num_sms, cudaStream_t stream) {
  const int grid = num_sms * 8, block = 256;
  if (in_bf16 && grad_bf16)
    normalize_bwd_kernel<true, true><<<grid, block, 0, stream>>>(x, inv_norm, dxhat, dx, rows, D / 8);
  else if (in_bf16)
    normalize_bwd_kernel<true, false><<<grid, block, 0, stream>>>(x, inv_norm, dxhat, dx, rows, D / 8);
  else if (grad_bf16)
    normalize_bwd_kernel<false, true><<<grid, block, 0, stream>>>(x, inv_norm, dxhat, dx, rows, D / 8);
  else
    normalize_bwd_kernel<false, false><<<grid, block, 0, stream>>>(x, inv_norm, dxhat, dx, rows, D / 8);
  return static_cast<int>(cudaGetLastError());
}

int launch_scale(const void* src, void* dst, int is_bf16, const float* g, size_t nbytes, int num_sms,
                 cudaStream_t stream) {
  const int aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0;
  scale_kernel<<<num_sms * 4, 256, 0, stream>>>(src, dst, is_bf16, g, nbytes, aligned);
  return static_cast<int>(cudaGetLastError());
}

int launch_allreduce_scalars(const float* saved, const float* g, float* mailbox_local, const float* const* mailboxes_dev,
                             unsigned int* const* signal_ptrs_dev, const volatile unsigned int* flags_local, int world,
                             unsigned int value, float* dt_prime, float* dbias, int dtp_f64,
                             unsigned long long timeout_ns, DebugRecord* dbg, cudaStream_t stream) {
  allreduce_scalars_kernel<<<1, 32, 0, stream>>>(saved, g, mailbox_local, mailboxes_dev, signal_ptrs_dev, flags_local,
                                                 world, value, dt_prime, dbias, dtp_f64, timeout_ns, dbg);
  return static_cast<int>(cudaGetLastError());
}

// fmaxf returns the non-NaN operand, so NaN -> 0 and the result is in [0, 1]
__global__ void clamp_weights_kernel(const float* src_a, float* dst_a, int na, const float* src_b, float* dst_b,
                                     int nb) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < na + nb; i += gridDim.x * blockDim.x) {
    const float* src = (i < na) ? src_a : src_b;
    const int k = (i < na) ? i : i - na;
    (i < na ? dst_a : dst_b)[k] = (src != nullptr) ? fminf(fmaxf(src[k], 0.f), 1.f) : 1.f;
  }
}

int launch_clamp_weights(const float* src_a, float* dst_a, int na, const float* src_b, float* dst_b, int nb,
                         cudaStream_t stream) {
  const int n = na + nb;
  const int blocks = (n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024;
  clamp_weights_kernel<<<blocks > 0 ? blocks : 1, 256, 0, stream>>>(src_a, dst_a, na, src_b, dst_b, nb);
  return static_cast<int>(cudaGetLastError());
}

int launch_metrics_finalize(const MetricsArgs& a, cudaStream_t stream) {
  metrics_finalize_kernel<<<1, kMetricsThreads, 0, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

int launch_metrics_finalize_labels(const MetricsArgs& a, const LabelSetArgs& l, cudaStream_t stream) {
  metrics_finalize_labels_kernel<<<1, kMetricsThreads, 0, stream>>>(a, l);
  return static_cast<int>(cudaGetLastError());
}

int launch_sample_loss_finalize(const SampleLossArgs& a, cudaStream_t stream) {
  sample_loss_finalize_kernel<<<1, kSampleLossThreads, 0, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

int launch_topk_finalize(const TopKArgs& a, cudaStream_t stream) {
  topk_finalize_kernel<<<1, kTopKThreads, 0, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

int launch_topk_finalize_labels(const TopKArgs& a, const LabelSetArgs& l, cudaStream_t stream) {
  topk_finalize_labels_kernel<<<1, kTopKThreads, 0, stream>>>(a, l);
  return static_cast<int>(cudaGetLastError());
}

int launch_signal_flags(unsigned int* const* flag_ptrs_dev, int n, unsigned int value, cudaStream_t stream) {
  signal_flags_kernel<<<1, 32, 0, stream>>>(flag_ptrs_dev, n, value);
  return static_cast<int>(cudaGetLastError());
}

int launch_wait_flags(const volatile unsigned int* flags, int n, unsigned int value, unsigned long long timeout_ns,
                      DebugRecord* dbg, cudaStream_t stream) {
  wait_flags_kernel<<<1, 32, 0, stream>>>(flags, n, value, timeout_ns, dbg);
  return static_cast<int>(cudaGetLastError());
}

static int launch_distill_opts(int cluster, const CUtensorMap* tmA0, const CUtensorMap* tmB0, const CUtensorMap* tmA1,
                               const CUtensorMap* tmB1, const CUtensorMap* tmG, const KernelParams& p, int num_sms,
                               cudaStream_t stream) {
  switch (cluster) {
    case 4: return launch_impl<kModeDistillOpts, kDistillStages, 4>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    case 2: return launch_impl<kModeDistillOpts, kDistillStages, 2>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    default: return launch_impl<kModeDistillOpts, kDistillStages, 1>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
  }
}

}  // namespace siglip

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

template <int kMode, int kStagesT>
struct Cfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;            // 16 KiB
  static constexpr int kBBytes = kTileN * kBlockK * 2;             // 16 KiB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = kStagesT;
  static constexpr int kStagingBytes = (kMode == kModeLoss) ? kNumEpiWarps * kStagingBytesPerWarp : 0;
  static constexpr int kSmemBytes =
      kStages * kStageBytes + kStagingBytes + 1024 /*barriers, reduction*/ + 1024 /*alignment slack*/;
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

// Fast path: every z of the slab is < kFastZ, so e = exp(z) < 2^-6 and both sigma(z) = e / (1 + e) and log1p(e) are
// evaluated by their alternating series on the FMA pipe (truncation < 3.4e-6 relative at the edge of the path, < 1e-8
// for the z ~ -10 of a SigLIP batch; the tolerance is 1e-3). One MUFU (ex2) per element instead of two: the epilogue
// is bound by the MUFU and FMA pipes.
__device__ __forceinline__ void loss_slab_fast(const float* v, float tl, float bl, int col0, bool store_g,
                                               const GStore& gst, float gscale, float& acc_sp, float& acc_g,
                                               float& acc_gs) {
  uint32_t packed[8];
  float a_sp = 0.f, a_g = 0.f, a_gs = 0.f;
  float g_prev = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float s = v[i];
    const float e = ex2_approx(fmaf(s, tl, bl));        // exp(z), z < kFastZ
    // sigma is produced already multiplied by the power-of-two scale of the 16-bit operand (exact), and the two sums
    // that use it are un-scaled once per slab
    float q = fmaf(e, gscale, -gscale);                  // S sigma(z) / e = S (1 - e + e^2)  [- e^3 < 3.8e-6 dropped]
    q = fmaf(e, q, gscale);
    const float g = e * q;                               // S sigma(z)
    float l = fmaf(e, 0.33333334f, -0.5f);               // log1p(e) / e = 1 - e/2 + e^2/3    [- e^3/4 < 1e-6 dropped]
    l = fmaf(e, l, 1.0f);
    a_sp = fmaf(e, l, a_sp);
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
template <bool kMask>
__device__ __forceinline__ void loss_slab(const float* v, float t, float b, int row_lo, int col0, int c_lo, int nrows,
                                          int ncols, bool store_g, const GStore& gst, float gscale, float* g_diag,
                                          bool on_diag, float& acc_sp, float& acc_g, float& acc_gs) {
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
        g_store = 0.f;                                 // the 16-bit operand carries negatives only
        if (store_g && valid) g_diag[row] = g;
      }
      sp = valid ? sp : 0.f;
      g = valid ? g : 0.f;
      g_store = valid ? g_store : 0.f;
    }
    acc_sp += sp;
    acc_g += g;
    acc_gs = fmaf(g, s, acc_gs);
    if (i & 1)
      packed[2 * (i >> 2) + ((i >> 1) & 1)] = pack_16x2<true>(g_prev, g_store * gscale);
    else
      g_prev = g_store * gscale;
  }
  if (store_g) store_g_slab(gst, col0, packed);
}

// Epilogue of the out kernel: one row of the fragment (h = 0: row_lo, 1: row_lo + 8), 16 column pairs.
//   val = scale * (acc * acc_scale + fix * x[row, col]) (+ add_src[row, col]);  written as fp32 or bf16
// parts / nparts: owner of a split tile — the other K-slices' fp32 partials (float4 j of this thread's fragment at
// parts[j * 256], slices part_stride apart) are added to acc first, in slice order. (Read here instead of being added
// into the accumulator registers: a non-wgmma write to them makes ptxas serialise every wgmma of the kernel.)
// All global loads of a group of four column pairs are issued before its stores: the stores may alias the loads as far
// as the compiler knows, and a load -> store -> load chain exposes one L2 round trip per pair.
__device__ __forceinline__ void out_row(const float (&acc)[64], int h, float scale, int row, int col0, int c_lo,
                                       const Problem& pr, float fix, const float4* parts = nullptr, int nparts = 0,
                                       size_t part_stride = 0) {
  if (row >= pr.M) return;
  const float as = pr.acc_scale;   // undoes the power-of-two scaling of the fp16 operands (1 for bf16)
  const float xs = (pr.fix_mat_scale != 0.f) ? pr.fix_mat_scale : 1.0f;
  const float fixs = fix * xs;
  const __nv_bfloat16* xrow = pr.fix_mat ? pr.fix_mat + static_cast<long long>(row) * pr.ldx : nullptr;
  const float* arow = pr.add_src ? pr.add_src + static_cast<long long>(row) * pr.ld_add : nullptr;
#pragma unroll
  for (int jb = 0; jb < 4; ++jb) {
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
// Mainloop of one consumer warpgroup: acc (+)= A[its 64 rows] * B[128 columns]^T over k-blocks [kb0, kb1), operands
// from the shared-memory ring. One k block = 4 wgmma's; the stage of the previous k block is handed back (to every CTA
// of the cluster that multicasts into it) once wgmma.wait_group says its MMAs have finished reading it.
// -------------------------------------------------------------------------------------------------
template <int kType, int kTA, int kTB, int kCS, int kStageBytes>
__device__ __forceinline__ void mma_loop(float (&acc)[64], int kb0, int kb1, int& stage, uint32_t& phase, int nstages,
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
  for (int i = 0; i < 64; ++i) acc_fence(acc[i]);
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(full0 + 8u * static_cast<uint32_t>(stage), phase, dbg, 3, t, kb, 0, waited);
    const uint64_t so = static_cast<uint64_t>(stage) * static_cast<uint64_t>(kStageBytes >> 4);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / kMmaK; ++k) {
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
  for (int i = 0; i < 64; ++i) acc_fence(acc[i]);
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

// -------------------------------------------------------------------------------------------------
// The kernel
// -------------------------------------------------------------------------------------------------
// kF8: the out kernel of the 8-bit measurement path (its own instantiation: the extra fp32 result registers of
// mma_loop_f8 would otherwise cost the production kernels spills).
template <int kMode, int kStagesT, int kCS, bool kF8 = false>
__global__ void __launch_bounds__(kNumThreads, 1)
siglip_gemm_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmB0,
                   const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmB1,
                   const __grid_constant__ CUtensorMap tmG, const __grid_constant__ KernelParams p) {
  using C = Cfg<kMode, kStagesT>;
  static_assert(kCS == 1 || kCS == 2 || kCS == 4, "clusters of 1, 2 or 4 CTAs");
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
    const uint64_t pol_a = (kMode == kModeLoss) ? pol_b : l2_policy_evict_normal();
    for (int t = cluster_id; t < total_tiles; t += num_clusters) {
      const TileCoord tc = decode_tile<kCS>(p, t, static_cast<int>(crank));
      const Problem& pr = p.prob[tc.prob];
      const CUtensorMap* tmA = tc.prob ? &tmA1 : &tmA0;
      const CUtensorMap* tmB = tc.prob ? &tmB1 : &tmB0;
      const int m_idx = tc.m_blk * kBlockM;
      const int n_idx = tc.n_blk * kTileN;
      // elements per 128-byte swizzle row: 64 16-bit values, or 128 8-bit ones (fp8 measurement path, K-major only)
      const int kblk = (pr.ab_f16 == 2) ? 2 * kBlockK : kBlockK;
      const int num_kb = (pr.K + kblk - 1) / kblk;
      const int a_mn = pr.a_mn, b_mn = pr.b_mn;
      int kb0, kb1;
      item_k_range(p, tc, num_kb, kb0, kb1);
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
            constexpr int kRows = kTileN / kCS;                     // box {64 k, kRows rows}
            load_b(sB + crank * (kRows * 128), k_idx, n_idx + static_cast<int>(crank) * kRows);
          } else if constexpr (kCS == 4) {
            // boxes {64 columns, 32 k}: CTA r fetches k half (r & 1) of the 64-column block (r >> 1)
            const int h = static_cast<int>(crank >> 1), kh = static_cast<int>(crank & 1u);
            load_b(sB + h * 8192 + kh * 4096, n_idx + 64 * h, k_idx + 32 * kh);
          } else {
#pragma unroll
            for (int h = static_cast<int>(crank) * (2 / kCS); h < (static_cast<int>(crank) + 1) * (2 / kCS); ++h)
              load_b(sB + h * 8192, n_idx + 64 * h, k_idx);         // boxes {64 columns, 64 k}
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
    const float bias = (kMode == kModeLoss) ? *p.bias : 0.f;
    // loss kernel: z = t_eff * acc + b with t_eff = t * s_scale (the accumulator is 2^8 <img, txt> for fp16 x 16 operands)
    const float s_scale = (kMode == kModeLoss && p.s_scale != 0.f) ? p.s_scale : 1.0f;
    const float t_eff = t_exact * s_scale;
    const float tl = t_eff * kLog2e, bl = bias * kLog2e;
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
    float acc[64];
    float acc8[kF8 ? 64 : 1];   // result of the 8-bit mainloop (see mma_loop_f8)
    for (int t = cluster_id; t < total_tiles; t += num_clusters) {
      const TileCoord tc = decode_tile<kCS>(p, t, static_cast<int>(crank));
      const Problem& pr = p.prob[tc.prob];
      const int row0 = tc.m_blk * kBlockM;            // first row of this CTA's block
      const int col_base = tc.n_blk * kTileN;
      const int row_lo = row0 + r_lo;                 // global rows of this thread: row_lo, row_lo + 8
      const bool fp8 = (pr.ab_f16 == 2);
      const int num_kb = (pr.K + (fp8 ? 2 * kBlockK : kBlockK) - 1) / (fp8 ? 2 * kBlockK : kBlockK);
      int kb0, kb1;
      item_k_range(p, tc, num_kb, kb0, kb1);
      {
        // K-major: 8-row groups 1024 B apart (SBO), K advance 32 B inside the swizzle row (16 16-bit or 32 8-bit values).
        // MN-major: 64-element MN blocks 8192 B apart (LBO), 8-k groups 1024 B apart (SBO), K advance 16 rows.
        // This warpgroup's 64 A rows start 8192 B into the A tile in both layouts.
        const uint32_t a_lbo = pr.a_mn ? 8192u : 16u, b_lbo = pr.b_mn ? 8192u : 16u;
        const uint32_t a_adv = pr.a_mn ? (kMmaK * 128u) >> 4 : 32u >> 4;
        const uint32_t b_adv = pr.b_mn ? (kMmaK * 128u) >> 4 : 32u >> 4;
        const uint64_t adesc0 = make_smem_desc_sw128(smem_base + static_cast<uint32_t>(wg) * 8192u, a_lbo, 1024u);
        const uint64_t bdesc0 = make_smem_desc_sw128(smem_base + C::kABytes, b_lbo, 1024u);
#define SIGLIP_MMA_LOOP(T, TA, TB)                                                                                  \
  mma_loop<T, TA, TB, kCS, C::kStageBytes>(acc, kb0, kb1, stage, phase, C::kStages, adesc0, bdesc0, a_adv, b_adv, \
                                           full0, empty0, lane, p.dbg, t, w_full_p)
        const int sel = pr.a_mn * 2 + pr.b_mn;
        if (fp8) {
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

      if constexpr (kMode == kModeLoss) {
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
#pragma unroll
        for (int c = 0; c < kTileN / 32; ++c) {
          const float* v = acc + 16 * c;
          const int col0 = col_base + 32 * c;
          // Only the 16x32 slabs that touch the diagonal of a diagonal block hold positive pairs, and only the slabs
          // that cross the matrix border of an edge block need masking; every other slab takes the fast path like
          // the rest of the matrix.
          const bool slab_diag = diag && (gst.row0 < col0 + 32) && (col0 < gst.row0 + 16);
          const bool slab_edge = edge && ((gst.row0 + 16 > pr.M) || (col0 + 32 > pr.N));
          if (!slab_edge && !slab_diag) {
            // z is monotone in s (t > 0): the slab is "all very negative" iff max s is
            float smax = v[0];
#pragma unroll
            for (int j = 1; j < 16; ++j) smax = fmaxf(smax, v[j]);
            const bool fast = __all_sync(0xffffffffu, fmaf(smax, t_eff, bias) < kFastZ);
            if (fast)
              loss_slab_fast(v, tl, bl, col0, sg, gst, p.g_scale, acc_sp, acc_g, acc_gs);
            else
              loss_slab<false>(v, t_eff, bias, row_lo, col0, c_lo, pr.M, pr.N, sg, gst, p.g_scale, p.g_diag, false,
                               acc_sp, acc_g, acc_gs);
          } else {
            loss_slab<true>(v, t_eff, bias, row_lo, col0, c_lo, pr.M, pr.N, sg, gst, p.g_scale, p.g_diag, slab_diag,
                            acc_sp, acc_g, acc_gs);
          }
        }
        kahan_add(s_sp, c_sp, acc_sp);
        kahan_add(s_g, c_g, acc_g);
        kahan_add(s_gs, c_gs, acc_gs);
      } else {
        const float scale = t_exact * p.inv_b * (p.grad_out != nullptr ? *p.grad_out : 1.0f);
        const float fix0 = (pr.fix_vec != nullptr && row_lo < pr.M) ? pr.fix_vec[row_lo] : 0.f;
        const float fix1 = (pr.fix_vec != nullptr && row_lo + 8 < pr.M) ? pr.fix_vec[row_lo + 8] : 0.f;
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
          out_row(acc8, 0, scale, row_lo, col_base, c_lo, pr, fix0);
          out_row(acc8, 1, scale, row_lo + 8, col_base, c_lo, pr, fix1);
        } else if (tc.part < 0) {
          out_row(acc, 0, scale, row_lo, col_base, c_lo, pr, fix0);
          out_row(acc, 1, scale, row_lo + 8, col_base, c_lo, pr, fix1);
        } else {
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
            out_row(acc, 0, scale, row_lo, col_base, c_lo, pr, fix0, ws, p.sk_parts - 1, part_stride);
            out_row(acc, 1, scale, row_lo + 8, col_base, c_lo, pr, fix1, ws, p.sk_parts - 1, part_stride);
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
    if constexpr (kMode == kModeLoss) {
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
            const float lo = fminf(fmaxf(__uint_as_float(w[q] << 16) * sc, -65504.f), 65504.f);
            const float hi = fminf(fmaxf(__uint_as_float(w[q] & 0xffff0000u) * sc, -65504.f), 65504.f);
            o[q] = pack_16x2<true>(lo, hi);
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

// fp16(v * scale), clamped to the fp16 range: the operand format of the fp32-input path
__device__ __forceinline__ void store8_f16(void* base, size_t idx8, const float (&v)[8], float scale) {
  uint32_t o[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float lo = fminf(fmaxf(v[2 * q] * scale, -65504.f), 65504.f);
    const float hi = fminf(fmaxf(v[2 * q + 1] * scale, -65504.f), 65504.f);
    o[q] = pack_16x2<true>(lo, hi);
  }
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

template <int kMode, int kStages, int kCS, bool kF8 = false>
int launch_impl(const CUtensorMap* tmA0, const CUtensorMap* tmB0, const CUtensorMap* tmA1, const CUtensorMap* tmB1,
                const CUtensorMap* tmG, const KernelParams& p, int num_sms, cudaStream_t stream) {
  using C = Cfg<kMode, kStages>;
  auto kern = siglip_gemm_kernel<kMode, kStages, kCS, kF8>;
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
    pr.tiles_n = (pr.N + kTileN - 1) / kTileN;
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
  if (kMode == kModeOut && p.sk_request != 0 && p.sk_ws != nullptr && clusters > 1) {
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
  if (clusters > total_tiles) clusters = total_tiles;
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

#define SIGLIP_LAUNCH(MODE, ST, CS) \
  return launch_impl<MODE, ST, CS>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream)

#define SIGLIP_LAUNCH_STAGES(MODE, CS)   \
  do {                                   \
    if (stages == 4) SIGLIP_LAUNCH(MODE, 4, CS); \
    SIGLIP_LAUNCH(MODE, 6, CS);          \
  } while (0)

int launch_gemm(int cta_group, int mode, int stages, int mcast, const CUtensorMap* tmA0, const CUtensorMap* tmB0,
                const CUtensorMap* tmA1, const CUtensorMap* tmB1, const CUtensorMap* tmG, const KernelParams& p,
                int num_sms, cudaStream_t stream) {
  if (stages <= 0) stages = default_stages(mode);
  if (mode == kModeOut && p.prob[0].ab_f16 == 2) {   // 8-bit measurement path: K-major, no multicast, no split-K
    if (cluster_size(cta_group, mcast) == 2)
      return launch_impl<kModeOut, 6, 2, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
    return launch_impl<kModeOut, 6, 1, true>(tmA0, tmB0, tmA1, tmB1, tmG, p, num_sms, stream);
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

int launch_signal_flags(unsigned int* const* flag_ptrs_dev, int n, unsigned int value, cudaStream_t stream) {
  signal_flags_kernel<<<1, 32, 0, stream>>>(flag_ptrs_dev, n, value);
  return static_cast<int>(cudaGetLastError());
}

int launch_wait_flags(const volatile unsigned int* flags, int n, unsigned int value, unsigned long long timeout_ns,
                      DebugRecord* dbg, cudaStream_t stream) {
  wait_flags_kernel<<<1, 32, 0, stream>>>(flags, n, value, timeout_ns, dbg);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace siglip

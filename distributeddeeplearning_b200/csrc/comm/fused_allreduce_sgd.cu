// Fused gradient allreduce + cast/scale + SGD-momentum update over NVLink peer / NVLS multicast
// memory — the native replacement for the reference's Horovod path
//   hvd.DistributedOptimizer: per-parameter allreduce_async_ -> fusion buffer -> ncclAllReduce ->
//   div_(size) -> optimizer.step() (161 x add_/mul_/add_)           (SURVEY.md X2, K12-K16, K19)
//
// One kernel per gradient bucket does, with NO NCCL call and NO separate optimizer kernel:
//   (wire=bf16 only) cast-and-scale this rank's fp32 gradients into the symmetric bf16 staging
//                    buffer and clear the fp32 accumulators                      [K13]
//   barrier-in       every rank's gradients for this bucket are complete
//   reduce-scatter   rank r owns slice r: multimem.ld_reduce (in-switch NVLS reduction) or
//                    8 peer loads over NVLink (P2P fallback)                    [K14]
//   update           g/N (+wd*w), momentum, w -= lr*m on the fp32 master slice   [K15]
//   all-gather       updated fp32 weights AND their bf16 compute copy are written to every
//                    replica with multimem.st (or 8 peer stores)                 [K14/K16]
//   clear            the reader of a gradient vector zeroes it on every replica   [K12]
//   barrier-out      (last bucket of the step only) every peer's stores have landed
//
// Cross-rank barriers are per-block flag exchanges in the symmetric signal pad with
// st.release.sys / ld.acquire.sys, epochs kept in device memory (CUDA-graph safe) and a bounded
// spin that raises a device-side error flag instead of hanging (SURVEY.md 5.3).
#include "../common.cuh"
#include "comm.h"

namespace ddl {

// ------------------------------------------------------------------------------------------
// multimem / sys-scope primitives
// ------------------------------------------------------------------------------------------
DDL_DEVICE float4 multimem_ld_reduce_f32x4(uint64_t mc_addr) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc_addr) : "memory");
  return v;
}
// 8 bf16 values reduced with fp32 accumulation inside the switch
DDL_DEVICE uint4 multimem_ld_reduce_bf16x8(uint64_t mc_addr) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc_addr) : "memory");
  return v;
}
DDL_DEVICE void multimem_st_f32x4(uint64_t mc_addr, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
DDL_DEVICE void multimem_st_u32x2(uint64_t mc_addr, const uint2& v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.bf16x2 [%0], {%1,%2};"
               :: "l"(mc_addr), "r"(v.x), "r"(v.y) : "memory");
}
DDL_DEVICE void multimem_st_u32x4(uint64_t mc_addr, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};"
               :: "l"(mc_addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
DDL_DEVICE float4 ld_peer_f32x4(uint64_t addr) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(addr) : "memory");
  return v;
}
DDL_DEVICE uint4 ld_peer_u32x4(uint64_t addr) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(addr) : "memory");
  return v;
}
DDL_DEVICE void st_peer_f32x4(uint64_t addr, const float4& v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
DDL_DEVICE void st_peer_u32x2(uint64_t addr, const uint2& v) {
  asm volatile("st.global.v2.u32 [%0], {%1,%2};" :: "l"(addr), "r"(v.x), "r"(v.y) : "memory");
}
DDL_DEVICE void st_peer_u32x4(uint64_t addr, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
DDL_DEVICE void st_release_sys(uint64_t addr, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(addr), "r"(v) : "memory");
}
DDL_DEVICE uint32_t ld_acquire_sys(uint64_t addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}

// ------------------------------------------------------------------------------------------
// block-level cross-rank barrier
// ------------------------------------------------------------------------------------------
// Signal pad layout (uint32), identical on every rank:  pad[channel][block][src_rank].
// Block b of rank r stores `epoch` into pad[ch][b][r] of EVERY rank, then waits until its own
// pad[ch][b][*] all reached `epoch`.  Epochs only grow, so a late reader never misses one.
// The block-uniform verdict lives in a shared flag indexed by the epoch's parity: a kernel issues at most two barriers,
// with consecutive epochs, so the thread that races ahead into the second barrier resets the OTHER slot while stragglers
// still read the first one (compute-sanitizer racecheck flagged the single-flag version: profiles/sanitizer.md).
DDL_DEVICE bool block_barrier(const CommCtx& c, int channel, uint32_t epoch) {
  __shared__ int s_timed_out2[2];
  int& s_timed_out = s_timed_out2[epoch & 1u];
  if (threadIdx.x == 0) s_timed_out = 0;
  __syncthreads();
  if (threadIdx.x < static_cast<unsigned>(c.world)) {
    const int peer = threadIdx.x;
    const uint64_t slot = (static_cast<uint64_t>(channel) * kMaxCommBlocks + blockIdx.x) * kMaxWorld;
    __threadfence_system();
    st_release_sys(c.peer_base[peer] + c.flag_off + (slot + c.rank) * 4u, epoch);
    const uint64_t mine = c.peer_base[c.rank] + c.flag_off + (slot + peer) * 4u;
    const uint64_t t0 = globaltimer_ns();
    uint32_t spins = 0;
    while (static_cast<int32_t>(ld_acquire_sys(mine) - epoch) < 0) {
      if ((++spins & 0x3ffu) == 0 && globaltimer_ns() - t0 > c.timeout_ns) {
        atomicExch(c.error_flag, 1u + static_cast<uint32_t>(peer));  // which peer never arrived
        s_timed_out = 1;
        break;
      }
    }
  }
  __syncthreads();
  // Block-uniform verdict.  A caller that sees `false` must NOT touch weights, momentum or gradients any more: a
  // peer's data is incomplete, and the host (FusedSGD.check_errors, polled by the trainers) aborts the job.
  return s_timed_out == 0;
}

// Each (channel, block) owns an epoch counter in local device memory; thread 0 bumps it by
// `n` and broadcasts the first new value.  Kept on the device so graph replays stay correct.
DDL_DEVICE uint32_t claim_epochs(const CommCtx& c, int channel, uint32_t n) {
  __shared__ uint32_t s_epoch;
  if (threadIdx.x == 0) {
    uint32_t* ctr = c.epoch_ctr + channel * kMaxCommBlocks + blockIdx.x;
    uint32_t e = *ctr;
    *ctr = e + n;
    s_epoch = e + 1;
  }
  __syncthreads();
  return s_epoch;
}

// ------------------------------------------------------------------------------------------
// SGD math (torch.optim.SGD semantics: wd added to grad, buf = mu*buf + (1-damp)*g,
// nesterov: g += mu*buf, w -= lr*g).  `first` = momentum buffer not initialised yet.
// ------------------------------------------------------------------------------------------
DDL_DEVICE void sgd_update(float& w, float& m, float g, const SgdHyper& h) {
  g = fmaf(h.weight_decay, w, g);
  if (h.momentum != 0.f) {
    m = h.first_step ? g : fmaf(h.momentum, m, (1.f - h.dampening) * g);
    g = h.nesterov ? fmaf(h.momentum, m, g) : m;
  }
  w = fmaf(-h.lr, g, w);
}

// ------------------------------------------------------------------------------------------
// world == 1: fused SGD + bf16 weight copy + gradient clear over one flat range
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) fused_sgd_local_kernel(float* __restrict__ w, float* __restrict__ g,
                                                              float* __restrict__ m,
                                                              __nv_bfloat16* __restrict__ wb,
                                                              const SgdHyper* __restrict__ hp, int64_t n4) {
  const SgdHyper h = *hp;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 gv = reinterpret_cast<float4*>(g)[i];
    float4 wv = reinterpret_cast<float4*>(w)[i];
    float4 mv = h.momentum != 0.f && !h.first_step ? reinterpret_cast<float4*>(m)[i] : make_float4(0, 0, 0, 0);
    const float s = h.grad_scale;
    sgd_update(wv.x, mv.x, gv.x * s, h);
    sgd_update(wv.y, mv.y, gv.y * s, h);
    sgd_update(wv.z, mv.z, gv.z * s, h);
    sgd_update(wv.w, mv.w, gv.w * s, h);
    reinterpret_cast<float4*>(w)[i] = wv;
    if (h.momentum != 0.f) reinterpret_cast<float4*>(m)[i] = mv;
    if (wb) reinterpret_cast<uint2*>(wb)[i] = make_uint2(pack_bf16x2(wv.x, wv.y), pack_bf16x2(wv.z, wv.w));
    reinterpret_cast<float4*>(g)[i] = make_float4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------------------------------
// world > 1: two-shot fused allreduce + SGD.  MC = NVLS multicast path, else P2P loads/stores.
// WIRE_BF16 = gradients travel as bfloat16 (the --fp16-allreduce analogue).
// ------------------------------------------------------------------------------------------
// ONESHOT (small buckets): every rank reduces the WHOLE bucket from all replicas (peer loads in rank order, so all
// ranks compute bit-identical sums) and updates only its own replica — no broadcast stores, one data phase instead of
// reduce-scatter + all-gather.  Two-shot (large buckets): rank r reduces slice r and broadcasts the new weights.
//
// Producer/consumer block identity (two-shot).  The cross-rank flag barrier pairs block b with block b of every
// peer, so every datum that crosses ranks must be produced, consumed and recycled by the SAME block index on all
// ranks.  The consumer of element e = start + slice*q + i*V (slice q, vector i) is thread (i mod nthreads) of rank
// q; therefore the bf16 staging prologue walks "for q: for i = tid; i < nvec; i += nthreads" (not a flat sweep of
// the bucket), and the gradient accumulators are recycled by their READER: after rank q has pulled vector i of all
// replicas it stores zeros to that vector of all replicas (multimem.st, or one peer store each) — the store carries a
// register dependence on the load's result, so it cannot overtake the read.  No block ever clears data a different
// block of a peer may still be reading, and no closing barrier is needed for the accumulators.
//
// Closing barrier.  What remains to be ordered is visibility of the peers' weight stores in MY replica before my
// next forward pass reads them.  Kernels of one rank run in stream order and every barrier-in executes a
// fence.sys (cumulative), so it is enough that the LAST bucket kernel of a step ends with a barrier
// (`b.closing`): when it completes locally, every block of every peer has fenced and signalled after the stores
// of all its earlier bucket kernels.  The other kernels return right after their data phase — they neither wait for
// the slowest peer a second time nor hold their SM slots while doing so.
template <bool MC, bool WIRE_BF16, bool ONESHOT>
__global__ void __launch_bounds__(512) fused_allreduce_sgd_kernel(CommCtx c, BucketArgs b) {
  const SgdHyper h = *b.hyper;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nthreads = gridDim.x * blockDim.x;
  const bool closing = ONESHOT || b.closing != 0;
  const uint32_t epoch = claim_epochs(c, b.channel, closing ? 2 : 1);
  const uint64_t self = c.peer_base[c.rank];
  constexpr int V = WIRE_BF16 ? 8 : 4;                  // elements per vector
  const int64_t slice = ONESHOT ? b.numel : b.numel / c.world;           // elements this rank reduces and updates
  const int64_t nvec = slice / V;
  const int nslices = ONESHOT ? 1 : c.world;

  auto debug_skew = [&]() {       // test hook: de-synchronise the blocks of a rank (and the ranks) on purpose
    if (c.debug_skew_ns != 0) {
      const uint64_t t0 = globaltimer_ns();
      const uint64_t wait = static_cast<uint64_t>((blockIdx.x + c.rank) % 4) * c.debug_skew_ns;
      while (globaltimer_ns() - t0 < wait) __nanosleep(200);
    }
  };
  if (WIRE_BF16) {
    debug_skew();
    // cast-and-scale prologue: fp32 accumulators -> symmetric bf16 staging, clear accumulators (local data only).
    // Same (slice, vector) -> thread mapping as the consumer loop below.
    const float s = h.grad_scale;
    for (int q = 0; q < nslices; ++q) {
      const int64_t sbase = b.start + slice * q;
      for (int64_t i = tid; i < nvec; i += nthreads) {
        const int64_t e = sbase + i * 8;
        float4* gp = reinterpret_cast<float4*>(self + c.grad_off + e * 4);
        float4 a = gp[0], d = gp[1];
        uint4 o = make_uint4(pack_bf16x2(a.x * s, a.y * s), pack_bf16x2(a.z * s, a.w * s),
                             pack_bf16x2(d.x * s, d.y * s), pack_bf16x2(d.z * s, d.w * s));
        *reinterpret_cast<uint4*>(self + c.stage_off + e * 2) = o;
        gp[0] = make_float4(0, 0, 0, 0);
        gp[1] = make_float4(0, 0, 0, 0);
      }
    }
  }
  if (!block_barrier(c, b.channel, epoch)) return;      // timeout: leave weights / momentum / gradients alone

  if (b.scalar_off != 0 && blockIdx.x == 0 && threadIdx.x < kScalarSlots / 4) {
    // piggy-backed metrics: every rank wrote its slot before this launch (stream order) and the barrier above made the
    // writes visible; peers overwrite their slot only after the closing barrier of this kernel (the engine puts the
    // scalars on the closing bucket).
    float4 acc = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int p = 0; p < kMaxWorld; ++p)
      if (p < c.world) {
        const float4 v = ld_peer_f32x4(c.peer_base[p] + b.scalar_off + threadIdx.x * 16);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    const float s = 1.0f / static_cast<float>(c.world);
    reinterpret_cast<float4*>(b.scalar_out)[threadIdx.x] = make_float4(acc.x * s, acc.y * s, acc.z * s, acc.w * s);
  }

  debug_skew();
  const int64_t base = ONESHOT ? b.start : b.start + slice * c.rank;     // (element offset in the arena)
  constexpr bool kSwitchReduce = MC && !ONESHOT;        // in-switch reduction order is not guaranteed identical
                                                        // for different requesters: one-shot sums peers itself
  // NVLink round trips are ~2-3 us: bytes in flight decide the bandwidth.  The in-switch path keeps U independent
  // 16-byte multimem.ld_reduce per thread outstanding, so a small grid (few SM slots taken from the backward pass
  // running next to this kernel) still fills the links; the peer-load path already has `world` loads per vector.
  constexpr int U = kSwitchReduce ? 4 : 1;
  for (int64_t i0 = tid; i0 < nvec; i0 += static_cast<int64_t>(U) * nthreads) {
    float gsum[U][V];
    uint32_t dep[U];                                     // 0, but data-dependent on the loads (orders the clears)
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + static_cast<int64_t>(u) * nthreads;
      dep[u] = 0;
      if (i >= nvec) continue;
      const int64_t e = base + i * V;
      if (WIRE_BF16) {
        if (kSwitchReduce) {
          const uint4 r = multimem_ld_reduce_bf16x8(c.mc_base + c.stage_off + e * 2);
          float2 p0 = unpack_bf16x2(r.x), p1 = unpack_bf16x2(r.y), p2 = unpack_bf16x2(r.z), p3 = unpack_bf16x2(r.w);
          gsum[u][0] = p0.x; gsum[u][1] = p0.y; gsum[u][2] = p1.x; gsum[u][3] = p1.y;
          gsum[u][V - 4] = p2.x; gsum[u][V - 3] = p2.y; gsum[u][V - 2] = p3.x; gsum[u][V - 1] = p3.y;
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) gsum[u][k] = 0.f;
          uint4 rr[kMaxWorld];
#pragma unroll
          for (int p = 0; p < kMaxWorld; ++p)
            if (p < c.world) rr[p] = ld_peer_u32x4(c.peer_base[p] + c.stage_off + e * 2);
#pragma unroll
          for (int p = 0; p < kMaxWorld; ++p)
            if (p < c.world) {
              float2 p0 = unpack_bf16x2(rr[p].x), p1 = unpack_bf16x2(rr[p].y), p2 = unpack_bf16x2(rr[p].z),
                     p3 = unpack_bf16x2(rr[p].w);
              gsum[u][0] += p0.x; gsum[u][1] += p0.y; gsum[u][2] += p1.x; gsum[u][3] += p1.y;
              gsum[u][V - 4] += p2.x; gsum[u][V - 3] += p2.y; gsum[u][V - 2] += p3.x; gsum[u][V - 1] += p3.y;
            }
        }
      } else {
        float4 r;
        if (kSwitchReduce) {
          r = multimem_ld_reduce_f32x4(c.mc_base + c.grad_off + e * 4);
        } else {
          float4 rr[kMaxWorld];
#pragma unroll
          for (int p = 0; p < kMaxWorld; ++p)
            if (p < c.world) rr[p] = ld_peer_f32x4(c.peer_base[p] + c.grad_off + e * 4);
          r = make_float4(0, 0, 0, 0);
#pragma unroll
          for (int p = 0; p < kMaxWorld; ++p)
            if (p < c.world) { r.x += rr[p].x; r.y += rr[p].y; r.z += rr[p].z; r.w += rr[p].w; }
        }
        asm volatile("and.b32 %0, %1, 0;" : "=r"(dep[u]) : "r"(__float_as_uint(r.x)));
        const float s = h.grad_scale;
        gsum[u][0] = r.x * s; gsum[u][1] = r.y * s; gsum[u][2] = r.z * s; gsum[u][3] = r.w * s;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + static_cast<int64_t>(u) * nthreads;
      if (i >= nvec) continue;
      const int64_t e = base + i * V;
      if (!WIRE_BF16 && !ONESHOT) {
        // recycle the accumulators of this vector on every replica (I am their only cross-rank reader)
        const float z = __uint_as_float(dep[u]);
        const float4 z4 = make_float4(z, z, z, z);
        if (MC) {
          multimem_st_f32x4(c.mc_base + c.grad_off + e * 4, z4);
        } else {
#pragma unroll
          for (int p = 0; p < kMaxWorld; ++p)
            if (p < c.world) st_peer_f32x4(c.peer_base[p] + c.grad_off + e * 4, z4);
        }
      }
      // fp32 master weights + momentum of my slice live in my own replica
      float wv[V], mv[V];
      const float4* wp = reinterpret_cast<const float4*>(self + c.weight_off + e * 4);
      float4* mp = reinterpret_cast<float4*>(b.momentum + e);
#pragma unroll
      for (int q = 0; q < V / 4; ++q) {
        float4 t = wp[q];
        wv[4 * q] = t.x; wv[4 * q + 1] = t.y; wv[4 * q + 2] = t.z; wv[4 * q + 3] = t.w;
        float4 m4 = (h.momentum != 0.f && !h.first_step) ? mp[q] : make_float4(0, 0, 0, 0);
        mv[4 * q] = m4.x; mv[4 * q + 1] = m4.y; mv[4 * q + 2] = m4.z; mv[4 * q + 3] = m4.w;
      }
#pragma unroll
      for (int k = 0; k < V; ++k) sgd_update(wv[k], mv[k], gsum[u][k], h);
#pragma unroll
      for (int q = 0; q < V / 4; ++q) {
        if (h.momentum != 0.f) mp[q] = make_float4(mv[4 * q], mv[4 * q + 1], mv[4 * q + 2], mv[4 * q + 3]);
        const float4 wn = make_float4(wv[4 * q], wv[4 * q + 1], wv[4 * q + 2], wv[4 * q + 3]);
        const uint2 wbn = make_uint2(pack_bf16x2(wn.x, wn.y), pack_bf16x2(wn.z, wn.w));
        const int64_t eo = e + 4 * q;
        if (ONESHOT) {
          *reinterpret_cast<float4*>(self + c.weight_off + eo * 4) = wn;
          *reinterpret_cast<uint2*>(self + c.wbf16_off + eo * 2) = wbn;
        } else if (MC) {
          multimem_st_f32x4(c.mc_base + c.weight_off + eo * 4, wn);
          multimem_st_u32x2(c.mc_base + c.wbf16_off + eo * 2, wbn);
        } else {
#pragma unroll
          for (int p = 0; p < kMaxWorld; ++p)
            if (p < c.world) {
              st_peer_f32x4(c.peer_base[p] + c.weight_off + eo * 4, wn);
              st_peer_u32x2(c.peer_base[p] + c.wbf16_off + eo * 2, wbn);
            }
        }
      }
    }
  }
  if (!closing) return;
  if (!block_barrier(c, b.channel, epoch + 1)) return;
  if (ONESHOT && !WIRE_BF16) {
    // one-shot: every rank read every replica; the identical flat mapping on all ranks makes block b the only
    // cross-rank reader of the vectors block b clears here
    const int64_t n4 = b.numel / 4;
    float4* gp = reinterpret_cast<float4*>(self + c.grad_off + b.start * 4);
    for (int64_t i = tid; i < n4; i += nthreads) gp[i] = make_float4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------------------------------
// plain in-place allreduce(sum) * scale on a symmetric fp32 / bf16 range (hvd.allreduce, sweep)
// ------------------------------------------------------------------------------------------
template <bool MC, bool BF16, bool ONESHOT>
__global__ void __launch_bounds__(512) allreduce_kernel(CommCtx c, int channel, uint64_t off, int64_t numel,
                                                       float scale) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nthreads = gridDim.x * blockDim.x;
  const uint32_t epoch = claim_epochs(c, channel, 2);
  if (!block_barrier(c, channel, epoch)) return;
  constexpr int V = BF16 ? 8 : 4;
  constexpr int ES = BF16 ? 2 : 4;
  const int64_t slice = ONESHOT ? numel : numel / c.world;
  const int64_t base = ONESHOT ? 0 : slice * c.rank;
  const int64_t nvec = slice / V;
  // one-shot reads every replica and writes only the local copy into the OUTPUT half
  // (off + numel*ES): inputs stay intact until the closing barrier.
  for (int64_t i = tid; i < nvec; i += nthreads) {
    const uint64_t bo = off + (base + i * V) * ES;
    uint4 out;
    if (BF16) {
      float a[8];
      if (MC) {
        uint4 r = multimem_ld_reduce_bf16x8(c.mc_base + bo);
        float2 p0 = unpack_bf16x2(r.x), p1 = unpack_bf16x2(r.y), p2 = unpack_bf16x2(r.z), p3 = unpack_bf16x2(r.w);
        a[0] = p0.x; a[1] = p0.y; a[2] = p1.x; a[3] = p1.y; a[4] = p2.x; a[5] = p2.y; a[6] = p3.x; a[7] = p3.y;
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = 0.f;
        uint4 rr[kMaxWorld];
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
          if (p < c.world) rr[p] = ld_peer_u32x4(c.peer_base[p] + bo);
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
          if (p < c.world) {
            float2 p0 = unpack_bf16x2(rr[p].x), p1 = unpack_bf16x2(rr[p].y), p2 = unpack_bf16x2(rr[p].z),
                   p3 = unpack_bf16x2(rr[p].w);
            a[0] += p0.x; a[1] += p0.y; a[2] += p1.x; a[3] += p1.y;
            a[4] += p2.x; a[5] += p2.y; a[6] += p3.x; a[7] += p3.y;
          }
      }
      out = make_uint4(pack_bf16x2(a[0] * scale, a[1] * scale), pack_bf16x2(a[2] * scale, a[3] * scale),
                       pack_bf16x2(a[4] * scale, a[5] * scale), pack_bf16x2(a[6] * scale, a[7] * scale));
    } else {
      float4 r;
      if (MC) {
        r = multimem_ld_reduce_f32x4(c.mc_base + bo);
      } else {
        float4 rr[kMaxWorld];
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
          if (p < c.world) rr[p] = ld_peer_f32x4(c.peer_base[p] + bo);
        r = make_float4(0, 0, 0, 0);
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
          if (p < c.world) { r.x += rr[p].x; r.y += rr[p].y; r.z += rr[p].z; r.w += rr[p].w; }
      }
      out = make_uint4(__float_as_uint(r.x * scale), __float_as_uint(r.y * scale), __float_as_uint(r.z * scale),
                       __float_as_uint(r.w * scale));
    }
    if (ONESHOT) {
      *reinterpret_cast<uint4*>(c.peer_base[c.rank] + bo + numel * ES) = out;
    } else if (MC) {
      multimem_st_u32x4(c.mc_base + bo, out);
    } else {
#pragma unroll
      for (int p = 0; p < kMaxWorld; ++p)
        if (p < c.world) st_peer_u32x4(c.peer_base[p] + bo, out);
    }
  }
  block_barrier(c, channel, epoch + 1);
}

// Bandwidth variant of the two-shot NVLS allreduce: 4 independent 16-byte multimem.ld_reduce per thread in flight
// before the matching multimem.st (NVLink round trips are ~2 us: bytes in flight decide the bandwidth).
template <bool BF16>
__global__ void __launch_bounds__(512) allreduce_mc_twoshot_kernel(CommCtx c, int channel, uint64_t off, int64_t numel,
                                                                   float scale) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nthreads = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const uint32_t epoch = claim_epochs(c, channel, 2);
  block_barrier(c, channel, epoch);
  constexpr int ES = BF16 ? 2 : 4;
  const int64_t slice_bytes = numel * ES / c.world;
  const uint64_t base = c.mc_base + off + static_cast<uint64_t>(slice_bytes) * c.rank;
  const int64_t n16 = slice_bytes / 16;
  constexpr int U = 4;
  for (int64_t i = tid; i < n16; i += U * nthreads) {
    if (BF16) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (i + u * nthreads < n16) v[u] = multimem_ld_reduce_bf16x8(base + (i + u * nthreads) * 16);
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (i + u * nthreads < n16) {
          if (scale != 1.0f) {
            float2 p;
            p = unpack_bf16x2(v[u].x); v[u].x = pack_bf16x2(p.x * scale, p.y * scale);
            p = unpack_bf16x2(v[u].y); v[u].y = pack_bf16x2(p.x * scale, p.y * scale);
            p = unpack_bf16x2(v[u].z); v[u].z = pack_bf16x2(p.x * scale, p.y * scale);
            p = unpack_bf16x2(v[u].w); v[u].w = pack_bf16x2(p.x * scale, p.y * scale);
          }
          multimem_st_u32x4(base + (i + u * nthreads) * 16, v[u]);
        }
    } else {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (i + u * nthreads < n16) v[u] = multimem_ld_reduce_f32x4(base + (i + u * nthreads) * 16);
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (i + u * nthreads < n16) {
          if (scale != 1.0f) { v[u].x *= scale; v[u].y *= scale; v[u].z *= scale; v[u].w *= scale; }
          multimem_st_f32x4(base + (i + u * nthreads) * 16, v[u]);
        }
    }
  }
  block_barrier(c, channel, epoch + 1);
}

// ------------------------------------------------------------------------------------------
// broadcast of a symmetric byte range from `root` to every replica (K16) and a pure barrier
// ------------------------------------------------------------------------------------------
template <bool MC>
__global__ void __launch_bounds__(512) broadcast_kernel(CommCtx c, int channel, uint64_t off, int64_t bytes,
                                                       int root) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nthreads = gridDim.x * blockDim.x;
  const uint32_t epoch = claim_epochs(c, channel, 2);
  block_barrier(c, channel, epoch);  // receivers are past their last use of the range
  if (c.rank == root) {
    const int64_t n16 = bytes / 16;
    const uint4* src = reinterpret_cast<const uint4*>(c.peer_base[c.rank] + off);
    for (int64_t i = tid; i < n16; i += nthreads) {
      uint4 v = src[i];
      if (MC) {
        multimem_st_u32x4(c.mc_base + off + i * 16, v);
      } else {
#pragma unroll
        for (int p = 0; p < kMaxWorld; ++p)
          if (p < c.world && p != root) st_peer_u32x4(c.peer_base[p] + off + i * 16, v);
      }
    }
  }
  block_barrier(c, channel, epoch + 1);
}

__global__ void barrier_kernel(CommCtx c, int channel) {
  const uint32_t epoch = claim_epochs(c, channel, 1);
  block_barrier(c, channel, epoch);
}

// all-gather of per-rank slices of a LOCAL (non-symmetric-source) fp32 buffer through the symmetric
// scratch range: used to assemble the sharded momentum for checkpoints.
template <bool MC>
__global__ void __launch_bounds__(512) allgather_slices_kernel(CommCtx c, int channel, const float* src,
                                                              uint64_t dst_off, int64_t start, int64_t numel) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int nthreads = gridDim.x * blockDim.x;
  const uint32_t epoch = claim_epochs(c, channel, 2);
  block_barrier(c, channel, epoch);
  const int64_t slice = numel / c.world;
  const int64_t base = start + slice * c.rank;
  for (int64_t i = tid; i < slice / 4; i += nthreads) {
    float4 v = reinterpret_cast<const float4*>(src + base)[i];
    const uint64_t o = dst_off + (base + i * 4) * 4;
    if (MC) {
      multimem_st_f32x4(c.mc_base + o, v);
    } else {
#pragma unroll
      for (int p = 0; p < kMaxWorld; ++p)
        if (p < c.world) st_peer_f32x4(c.peer_base[p] + o, v);
    }
  }
  block_barrier(c, channel, epoch + 1);
}

// ------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------
static inline int clamp_blocks(int blocks) {
  if (blocks < 1) blocks = 1;
  if (blocks > kMaxCommBlocks) blocks = kMaxCommBlocks;
  return blocks;
}

cudaError_t launch_fused_sgd_local(float* w, float* g, float* m, void* wb, const SgdHyper* hp, int64_t numel,
                                   int blocks, cudaStream_t stream) {
  if (numel % 4 != 0) return cudaErrorInvalidValue;
  fused_sgd_local_kernel<<<blocks < 1 ? 1 : blocks, 512, 0, stream>>>(w, g, m, static_cast<__nv_bfloat16*>(wb), hp,
                                                                     numel / 4);
  return cudaGetLastError();
}

cudaError_t launch_fused_allreduce_sgd(const CommCtx& c, const BucketArgs& b, bool use_mc, bool wire_bf16,
                                       int blocks, cudaStream_t stream) {
  if (b.numel % (static_cast<int64_t>(c.world) * 8) != 0) return cudaErrorInvalidValue;
  blocks = clamp_blocks(blocks);
  if (use_mc && c.mc_base == 0) return cudaErrorInvalidValue;
#define DDL_FUSED(MCV, WB, OS) fused_allreduce_sgd_kernel<MCV, WB, OS><<<blocks, 512, 0, stream>>>(c, b)
  if (b.oneshot) {
    if (wire_bf16) DDL_FUSED(false, true, true); else DDL_FUSED(false, false, true);
  } else if (use_mc) {
    if (wire_bf16) DDL_FUSED(true, true, false); else DDL_FUSED(true, false, false);
  } else {
    if (wire_bf16) DDL_FUSED(false, true, false); else DDL_FUSED(false, false, false);
  }
#undef DDL_FUSED
  return cudaGetLastError();
}

cudaError_t launch_allreduce(const CommCtx& c, int channel, uint64_t off, int64_t numel, bool bf16, float scale,
                             bool use_mc, bool oneshot, int blocks, cudaStream_t stream) {
  const int v = bf16 ? 8 : 4;
  if (numel % (static_cast<int64_t>(c.world) * v) != 0) return cudaErrorInvalidValue;
  blocks = clamp_blocks(blocks);
  if (use_mc && c.mc_base == 0) return cudaErrorInvalidValue;
#define DDL_AR(MC, BF, OS) allreduce_kernel<MC, BF, OS><<<blocks, 512, 0, stream>>>(c, channel, off, numel, scale)
  if (use_mc) {
    if (bf16) {
      if (oneshot) DDL_AR(true, true, true);
      else allreduce_mc_twoshot_kernel<true><<<blocks, 512, 0, stream>>>(c, channel, off, numel, scale);
    } else {
      if (oneshot) DDL_AR(true, false, true);
      else allreduce_mc_twoshot_kernel<false><<<blocks, 512, 0, stream>>>(c, channel, off, numel, scale);
    }
  } else {
    if (bf16) { if (oneshot) DDL_AR(false, true, true); else DDL_AR(false, true, false); }
    else      { if (oneshot) DDL_AR(false, false, true); else DDL_AR(false, false, false); }
  }
#undef DDL_AR
  return cudaGetLastError();
}

cudaError_t launch_broadcast(const CommCtx& c, int channel, uint64_t off, int64_t bytes, int root, bool use_mc,
                             int blocks, cudaStream_t stream) {
  if (bytes % 16 != 0) return cudaErrorInvalidValue;
  blocks = clamp_blocks(blocks);
  if (use_mc && c.mc_base != 0) broadcast_kernel<true><<<blocks, 512, 0, stream>>>(c, channel, off, bytes, root);
  else broadcast_kernel<false><<<blocks, 512, 0, stream>>>(c, channel, off, bytes, root);
  return cudaGetLastError();
}

cudaError_t launch_barrier(const CommCtx& c, int channel, cudaStream_t stream) {
  barrier_kernel<<<1, 32, 0, stream>>>(c, channel);
  return cudaGetLastError();
}

cudaError_t launch_allgather_slices(const CommCtx& c, int channel, const float* src, uint64_t dst_off,
                                    int64_t start, int64_t numel, bool use_mc, int blocks, cudaStream_t stream) {
  if (numel % (static_cast<int64_t>(c.world) * 4) != 0) return cudaErrorInvalidValue;
  blocks = clamp_blocks(blocks);
  if (use_mc && c.mc_base != 0)
    allgather_slices_kernel<true><<<blocks, 512, 0, stream>>>(c, channel, src, dst_off, start, numel);
  else
    allgather_slices_kernel<false><<<blocks, 512, 0, stream>>>(c, channel, src, dst_off, start, numel);
  return cudaGetLastError();
}

}  // namespace ddl

// Collectives of the data-parallel step fused into the kernels that need them, over NVLink peer
// memory (no NCCL on these paths):
//
//   * SyncBatchNormalization (tf2/resnet.py:54-60): the cross-replica sum of the per-channel
//     (sum x, sum x^2) -- and of (sum dz, sum dz*xhat) in the backward pass -- is a ONE-SHOT exchange
//     inside the finalize / coefficient kernel: every rank stores its [2C] doubles straight into every
//     peer's slot, releases a flag, waits for the R flags of its own slot and sums the R contributions
//     in rank order (bit-identical on every rank).  112 NCCL all-reduces per ResNet-50 step become
//     112 extra microseconds.
//   * tpu_cross_replica_concat (tf2/objective.py:92-127): the all-gather of the normalised embeddings
//     (and of the per-row log-sum-exp for the backward pass) as a push of this rank's rows into every
//     peer's gather region.
//
// All buffers live in ONE symmetric allocation per rank (same layout everywhere, peer base pointers
// in `peers[world]`): the caller passes byte offsets.  Ordering: data stores, __threadfence_system(),
// then a release store of the sequence number into the peer's flag word; the consumer polls its own
// flag words with acquire loads.  Sequence numbers live in device memory and are advanced by the
// kernels themselves, so the step can be captured in a CUDA graph and replayed; the word after each
// sequence number accumulates the nanoseconds this rank spent waiting for its peers.  Every spin is
// bounded: a protocol error traps after SPIN_TIMEOUT_NS instead of hanging the GPU.
#include "common.cuh"

namespace simclr {
namespace {

constexpr unsigned long long SPIN_TIMEOUT_NS = 20ull * 1000 * 1000 * 1000;

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
__device__ __forceinline__ void wait_flag(const unsigned long long* p, unsigned long long want, int tag) {
  unsigned long long t0 = 0; unsigned spins = 0;
  while (ld_acquire_sys(p) < want) {
    if ((++spins & 0x3ff) == 0) {
      const unsigned long long now = gtimer();
      if (t0 == 0) t0 = now;
      else if (now - t0 > SPIN_TIMEOUT_NS) {
        printf("simclr_b200 comm: peer flag timeout tag=%d want=%llu have=%llu\n", tag, want, ld_acquire_sys(p));
        __trap();
      }
    }
  }
}

struct Peers {
  void* const* bufs;     // [world] base pointers of the symmetric allocation (device array)
  int rank, world;
};

// One CTA.  Pushes `n` doubles to slot (seq % nslot), region `rank`, of every peer; returns (after a
// CTA barrier) with all `world` regions of the local slot complete.  `slot_doubles` = capacity of a region.
__device__ __forceinline__ const double* exchange_doubles(const Peers& P, const double* __restrict__ local, int n,
                                                          long long data_off, long long flag_off, int nslot,
                                                          long long slot_doubles, unsigned long long seq,
                                                          unsigned long long* __restrict__ wait_ns) {
  const int slot = (int)(seq % (unsigned long long)nslot);
  const long long region = ((long long)slot * P.world + P.rank) * slot_doubles;
  for (int r = 0; r < P.world; ++r) {
    double* dst = reinterpret_cast<double*>(reinterpret_cast<char*>(P.bufs[r]) + data_off) + region;
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = local[i];
  }
  __threadfence_system();
  __syncthreads();
  const unsigned long long t0 = threadIdx.x == 0 ? gtimer() : 0ull;
  if ((int)threadIdx.x < P.world) {
    unsigned long long* pf = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(P.bufs[threadIdx.x]) + flag_off) +
                             (long long)slot * P.world + P.rank;
    st_release_sys(pf, seq);
    const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(
        reinterpret_cast<const char*>(P.bufs[P.rank]) + flag_off) + (long long)slot * P.world + threadIdx.x;
    wait_flag(mine, seq, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) *wait_ns += gtimer() - t0;      // time this rank spent waiting for its peers (bench.py reports it)
  return reinterpret_cast<const double*>(reinterpret_cast<const char*>(P.bufs[P.rank]) + data_off) +
         (long long)slot * P.world * slot_doubles;
}

__global__ void __launch_bounds__(1024, 1)
bn_finalize_sync_kernel(Peers P, const double* __restrict__ sums, double count_local,
                        const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                        float* __restrict__ mm, float* __restrict__ mv, float* __restrict__ mean,
                        float* __restrict__ rstd, float* __restrict__ scale, float* __restrict__ shift, int C,
                        long long data_off, long long flag_off, int nslot, long long slot_doubles,
                        unsigned long long* __restrict__ seq_dev) {
  const unsigned long long seq = *seq_dev;
  const double* all = exchange_doubles(P, sums, 2 * C, data_off, flag_off, nslot, slot_doubles, seq, seq_dev + 1);
  const double count = count_local * P.world;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s0 = 0.0, s1 = 0.0;
    for (int r = 0; r < P.world; ++r) { s0 += __ldcg(all + r * slot_doubles + c); s1 += __ldcg(all + r * slot_doubles + C + c); }
    bn_finalize_channel(s0, s1, count, gamma, beta, eps, momentum, mm, mv, mean, rstd, scale, shift, c);
  }
  __syncthreads();
  if (threadIdx.x == 0) *seq_dev = seq + 1;
}

// coef = (k1, k2, k3) of dy = k1*dz + k2*y + k3 (bn.cu, bn_bwd_coef_kernel) from the GLOBAL sums;
// dgamma / dbeta are this replica's contributions (the gradient all-reduce sums them).
__global__ void __launch_bounds__(1024, 1)
bn_bwd_coef_sync_kernel(Peers P, const double* __restrict__ sums, double count_local,
                        const float* __restrict__ mean, const float* __restrict__ rstd,
                        const float* __restrict__ gamma, float* __restrict__ coef, float* __restrict__ dgamma,
                        float* __restrict__ dbeta, int C, long long data_off, long long flag_off, int nslot,
                        long long slot_doubles, unsigned long long* __restrict__ seq_dev) {
  const unsigned long long seq = *seq_dev;
  const double* all = exchange_doubles(P, sums, 2 * C, data_off, flag_off, nslot, slot_doubles, seq, seq_dev + 1);
  const double inv_count = 1.0 / (count_local * P.world);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s0 = 0.0, s1 = 0.0;
    for (int r = 0; r < P.world; ++r) { s0 += __ldcg(all + r * slot_doubles + c); s1 += __ldcg(all + r * slot_doubles + C + c); }
    const double r_ = rstd[c], mu = mean[c], g = gamma ? gamma[c] : 1.0;
    const double a = s0 * inv_count, b = s1 * inv_count;
    coef[c] = (float)(g * r_);
    coef[C + c] = (float)(-g * r_ * r_ * b);
    coef[2 * C + c] = (float)(g * r_ * (mu * r_ * b - a));
    if (dbeta) dbeta[c] = (float)sums[c];
    if (dgamma) dgamma[c] = (float)sums[C + c];
  }
  __syncthreads();
  if (threadIdx.x == 0) *seq_dev = seq + 1;
}

// All-gather by pushes: `chunk` bytes per rank (16-byte multiple) into region `rank` of every peer's
// gather area.  Several CTAs copy; the last one to finish publishes the flags and waits for the peers'.
// One region per channel (static addresses, so the consumers can sit in a captured graph): a rank
// may overwrite a peer's copy of step t only in step t+1, and it cannot get there before that peer
// has consumed step t -- every step ends with a collective over the gradients that needs all ranks.
__global__ void __launch_bounds__(256)
all_gather_push_kernel(Peers P, const uint4* __restrict__ src, long long chunk16, long long data_off,
                       long long flag_off, long long chunk_stride16, unsigned long long* __restrict__ seq_dev,
                       unsigned int* __restrict__ arrive) {
  const unsigned long long seq = *seq_dev;
  const long long region16 = (long long)P.rank * chunk_stride16;
  for (int r = 0; r < P.world; ++r) {
    uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<char*>(P.bufs[r]) + data_off) + region16;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < chunk16; i += (long long)gridDim.x * blockDim.x)
      dst[i] = src[i];
  }
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(arrive, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!last) return;
  __threadfence_system();
  const unsigned long long t0 = threadIdx.x == 0 ? gtimer() : 0ull;
  if ((int)threadIdx.x < P.world) {
    unsigned long long* pf = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(P.bufs[threadIdx.x]) + flag_off) + P.rank;
    st_release_sys(pf, seq);
    const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(
        reinterpret_cast<const char*>(P.bufs[P.rank]) + flag_off) + threadIdx.x;
    wait_flag(mine, seq, 2);
  }
  __syncthreads();
  if (threadIdx.x == 0) { *arrive = 0u; *seq_dev = seq + 1; seq_dev[1] += gtimer() - t0; }
}

}  // namespace
}  // namespace simclr

using namespace simclr;

extern "C" {

int simclr_comm_bn_finalize(const double* sums_local, double count_local, const float* gamma, const float* beta,
                            float eps, float momentum, float* moving_mean, float* moving_var, float* mean,
                            float* rstd, float* scale, float* shift, int64_t C, const void* peer_bufs_dev,
                            int rank, int world, int64_t data_off, int64_t flag_off, int nslot,
                            int64_t slot_bytes, void* seq_dev, void* stream) {
  SIMCLR_CHECK_ARG(sums_local && mean && rstd && scale && shift && peer_bufs_dev && seq_dev, "comm_bn_finalize: null pointer");
  SIMCLR_CHECK_ARG(C > 0 && count_local > 0 && world >= 1 && world <= 64 && rank >= 0 && rank < world && nslot >= 2,
                   "comm_bn_finalize: bad arguments");
  SIMCLR_CHECK_ARG(2 * C * 8 <= slot_bytes && slot_bytes % 16 == 0 && data_off % 16 == 0 && flag_off % 8 == 0,
                   "comm_bn_finalize: 2*C doubles (%lld) do not fit the exchange slot (%lld bytes)", (long long)(2 * C), (long long)slot_bytes);
  Peers P{reinterpret_cast<void* const*>(peer_bufs_dev), rank, world};
  bn_finalize_sync_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(
      P, sums_local, count_local, gamma, beta, eps, momentum, moving_mean, moving_var, mean, rstd, scale, shift, (int)C,
      (long long)data_off, (long long)flag_off, nslot, (long long)(slot_bytes / 8), (unsigned long long*)seq_dev);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_comm_bn_bwd_coef(const double* sums_local, double count_local, const float* mean, const float* rstd,
                            const float* gamma, float* coef, float* dgamma, float* dbeta, int64_t C,
                            const void* peer_bufs_dev, int rank, int world, int64_t data_off, int64_t flag_off,
                            int nslot, int64_t slot_bytes, void* seq_dev, void* stream) {
  SIMCLR_CHECK_ARG(sums_local && mean && rstd && coef && peer_bufs_dev && seq_dev, "comm_bn_bwd_coef: null pointer");
  SIMCLR_CHECK_ARG(C > 0 && count_local > 0 && world >= 1 && world <= 64 && rank >= 0 && rank < world && nslot >= 2,
                   "comm_bn_bwd_coef: bad arguments");
  SIMCLR_CHECK_ARG(2 * C * 8 <= slot_bytes && slot_bytes % 16 == 0 && data_off % 16 == 0 && flag_off % 8 == 0,
                   "comm_bn_bwd_coef: 2*C doubles do not fit the exchange slot");
  Peers P{reinterpret_cast<void* const*>(peer_bufs_dev), rank, world};
  bn_bwd_coef_sync_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(
      P, sums_local, count_local, mean, rstd, gamma, coef, dgamma, dbeta, (int)C, (long long)data_off,
      (long long)flag_off, nslot, (long long)(slot_bytes / 8), (unsigned long long*)seq_dev);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

int simclr_comm_all_gather(const void* src, int64_t nbytes, const void* peer_bufs_dev, int rank, int world,
                           int64_t data_off, int64_t flag_off, int64_t chunk_stride_bytes, void* seq_dev,
                           void* arrive_dev, void* stream) {
  SIMCLR_CHECK_ARG(src && peer_bufs_dev && seq_dev && arrive_dev, "comm_all_gather: null pointer");
  SIMCLR_CHECK_ARG(nbytes > 0 && nbytes % 16 == 0 && nbytes <= chunk_stride_bytes && chunk_stride_bytes % 16 == 0 &&
                   data_off % 16 == 0 && flag_off % 8 == 0 && aligned16(src),
                   "comm_all_gather: sizes/offsets must be 16-byte multiples (nbytes=%lld stride=%lld)", (long long)nbytes, (long long)chunk_stride_bytes);
  SIMCLR_CHECK_ARG(world >= 1 && world <= 64 && rank >= 0 && rank < world, "comm_all_gather: bad rank/world");
  Peers P{reinterpret_cast<void* const*>(peer_bufs_dev), rank, world};
  const long long chunk16 = nbytes / 16;
  long long grid = (chunk16 + 256 * 8 - 1) / (256 * 8);
  if (grid > 32) grid = 32;
  if (grid < 1) grid = 1;
  all_gather_push_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(
      P, (const uint4*)src, chunk16, (long long)data_off, (long long)flag_off, (long long)(chunk_stride_bytes / 16),
      (unsigned long long*)seq_dev, (unsigned int*)arrive_dev);
  SIMCLR_CHECK_LAUNCH();
  return SIMCLR_OK;
}

}  // extern "C"

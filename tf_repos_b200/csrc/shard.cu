// shard.cu -- routing helpers for the row-sharded embedding table (config 5: 1e9 rows over 8 GPUs).
//
// Not in the reference (its parameter server keeps each variable whole on one PS task, SURVEY.md 2.4).
// owner(id) = id % G, local row = id / G  (mod spreads the 13 always-present continuous-feature ids
// over the GPUs).  A rank de-duplicates its batch's ids (ctr_unique_segment), buckets the unique ids
// by owner (here), exchanges them with an NCCL all-to-all, the owners gather the rows (K1 gather
// kernels) and the rows come back the same way; gradients take the reverse route.
#include "common.cuh"

namespace ctr {

constexpr int MAX_G = 64;

__global__ void gather_scalar_kernel(const int32_t* __restrict__ ids, const float* __restrict__ W, int64_t N,
                                     int64_t n, float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t id = ids[i];
    out[i] = (id >= 0 && id < N) ? __ldg(W + id) : 0.f;
  }
}

// ---- composite keys: one sort gives bucket order, cache positions and the gradient segments -------------------
// key(id) = owner * Npad + local row, Npad = ceil(N / G).  Sorting the keys (ctr_unique_segment) orders the
// unique ids by (owner, id): the buckets of the id all-to-all are contiguous runs of `uniq`, an occurrence's cache
// position IS its `inverse` entry, and perm / seg_offsets already describe the gradient segments in cache order --
// no placement pass, no remap pass and no second sort.  Deterministic (no atomics decide an order).
__global__ void shard_keys_kernel(const int32_t* __restrict__ ids, int64_t n, int64_t N, int G, int32_t Npad,
                                  int32_t* __restrict__ keys, int32_t* __restrict__ oob) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    int64_t id = ids[i];
    if (id < 0 || id >= N) {
      if (oob) { if (atomicAdd(&oob[0], 1) == 0) oob[1] = (int32_t)id; }
      id = 0;
    }
    keys[i] = (int32_t)((id % G) * Npad + id / G);
  }
}

__global__ void __launch_bounds__(256)
shard_split_kernel(const int32_t* __restrict__ uniq, const int32_t* __restrict__ n_uniq, int64_t n_max, int32_t Npad,
                   int G, int32_t* __restrict__ counts, int32_t* __restrict__ local_ids) {
  __shared__ int32_t sh[MAX_G];
  if (threadIdx.x < G) sh[threadIdx.x] = 0;
  __syncthreads();
  const int64_t n = min((int64_t)n_uniq[0], n_max);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n; u += stride) {
    const int32_t key = uniq[u];
    const int o = key / Npad;
    local_ids[u] = key - o * Npad;
    atomicAdd(&sh[o], 1);          // integer counts: the result does not depend on the order
  }
  __syncthreads();
  if (threadIdx.x < G && sh[threadIdx.x]) atomicAdd(&counts[threadIdx.x], sh[threadIdx.x]);
}

static int lin_grid(int64_t n) {
  int64_t b = ceil_div64(n, 256);
  if (b < 1) b = 1;
  return (int)(b < (int64_t)sm_count() * 8 ? b : (int64_t)sm_count() * 8);
}

}  // namespace ctr

using namespace ctr;

extern "C" {

int ctr_shard_keys(const int32_t* ids, int64_t n, int64_t N, int G, int32_t* keys, int32_t* oob, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && N > 0 && G >= 1 && G <= MAX_G, CTR_ERR_INVALID_ARG, "ctr_shard_keys: bad n/N/G");
  const int64_t npad = (N + G - 1) / G;
  CTR_REQUIRE(npad * G <= 2147483647LL, CTR_ERR_UNSUPPORTED, "ctr_shard_keys: G*ceil(N/G) must fit int32");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(ids && keys, CTR_ERR_INVALID_ARG, "ctr_shard_keys: null buffer");
  shard_keys_kernel<<<lin_grid(n), 256, 0, as_stream(stream)>>>(ids, n, N, G, (int32_t)npad, keys, oob);
  CTR_LAUNCHED("ctr_shard_keys");
  return CTR_OK;
}

int ctr_shard_split(const int32_t* uniq_keys, const int32_t* n_uniq, int64_t n_max, int64_t N, int G, int32_t* counts,
                    int32_t* local_ids, ctr_stream_t stream) {
  CTR_REQUIRE(n_max >= 0 && N > 0 && G >= 1 && G <= MAX_G, CTR_ERR_INVALID_ARG, "ctr_shard_split: bad n_max/N/G");
  CTR_REQUIRE(uniq_keys && n_uniq && counts && local_ids, CTR_ERR_INVALID_ARG, "ctr_shard_split: null buffer");
  cudaStream_t st = as_stream(stream);
  CTR_REQUIRE(cudaMemsetAsync(counts, 0, G * sizeof(int32_t), st) == cudaSuccess, CTR_ERR_CUDA, "ctr_shard_split: memset failed");
  if (n_max == 0) return CTR_OK;
  shard_split_kernel<<<lin_grid(n_max), 256, 0, st>>>(uniq_keys, n_uniq, n_max, (int32_t)((N + G - 1) / G), G, counts, local_ids);
  CTR_LAUNCHED("ctr_shard_split");
  return CTR_OK;
}

int ctr_gather_scalar(const int32_t* ids, const float* W, int64_t N, int64_t n, float* out, ctr_stream_t stream) {
  CTR_REQUIRE(n >= 0 && N > 0, CTR_ERR_INVALID_ARG, "ctr_gather_scalar: bad args");
  if (n == 0) return CTR_OK;
  CTR_REQUIRE(ids && W && out, CTR_ERR_INVALID_ARG, "ctr_gather_scalar: null buffer");
  gather_scalar_kernel<<<lin_grid(n), 256, 0, as_stream(stream)>>>(ids, W, N, n, out);
  CTR_LAUNCHED("ctr_gather_scalar");
  return CTR_OK;
}

}  // extern "C"

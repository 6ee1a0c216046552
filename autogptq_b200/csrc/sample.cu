// Host side of next-token sampling (include/autogptq_b200.h: agb200_sample): argument checking and the cluster launch
// on the caller's stream.  Kernel: sample.cuh.
#include <cuda_runtime.h>

#include "host.h"
#include "sample.cuh"

static_assert(agb::kSampleMaxV == AGB200_SAMPLE_MAX_V, "sampler vocabulary limit");

template <int DT>
static int launch_sample(const agb::SampleParams& p, int B, cudaStream_t s) {
  constexpr auto kern = agb::sample_kernel<DT>;
  if (int rc = opt_in_smem<kern>(agb::kSampleSmemBytes)) return rc;
  return launch(kern, dim3(agb::kSampleCtas, B), dim3(agb::kSampleThreads), static_cast<size_t>(p.slice) * 4, s, false,
                dim3(agb::kSampleCtas, 1, 1), false, p);
}

extern "C" {

int agb200_sample(const void* logits, int64_t row_stride, int dtype, int B, int V, const float* temperature,
                  const int32_t* top_k, const float* top_p, const float* min_p, const uint64_t* seed,
                  const int64_t* counter, int64_t* tokens, void* stream) {
  if (!logits || !temperature || !top_k || !top_p || !min_p || !seed || !counter || !tokens)
    return failf(AGB200_EINVAL, "sample: null pointer argument");
  if (B < 1 || V < 1) return failf(AGB200_EINVAL, "sample: need B >= 1 and V >= 1 (got B=%d, V=%d)", B, V);
  if (row_stride < V)
    return failf(AGB200_EINVAL, "sample: row_stride %lld is below V=%d", static_cast<long long>(row_stride), V);
  if (dtype != AGB200_F16 && dtype != AGB200_BF16 && dtype != AGB200_F32)
    return failf(AGB200_ENOSUP, "sample: dtype %d; only AGB200_F16, AGB200_BF16 and AGB200_F32 are supported", dtype);
  if (V > AGB200_SAMPLE_MAX_V) return failf(AGB200_ENOSUP, "sample: V=%d; at most %d", V, AGB200_SAMPLE_MAX_V);
  if (B > 65535) return failf(AGB200_ENOSUP, "sample: B=%d rows; at most 65535", B);
  const int esize = dtype == AGB200_F32 ? 4 : 2;
  if (!aligned(logits, esize) || !aligned(temperature, 4) || !aligned(top_k, 4) || !aligned(top_p, 4) ||
      !aligned(min_p, 4) || !aligned(seed, 8) || !aligned(counter, 8) || !aligned(tokens, 8))
    return failf(AGB200_EINVAL, "sample: logits must be aligned to its element, the fp32 and int32 arrays to 4 bytes, "
                 "seed, counter and tokens to 8");
  agb::SampleParams p{};
  p.logits = logits;
  p.stride = row_stride;
  p.V = V;
  p.slice = static_cast<int>(align_up((V + agb::kSampleCtas - 1) / agb::kSampleCtas, 4));
  p.temperature = temperature;
  p.top_k = top_k;
  p.top_p = top_p;
  p.min_p = min_p;
  p.seed = seed;
  p.counter = counter;
  p.tokens = tokens;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == AGB200_F32) return launch_sample<2>(p, B, s);
  if (dtype == AGB200_BF16) return launch_sample<1>(p, B, s);
  return launch_sample<0>(p, B, s);
}

}  // extern "C"

// hll_estimate.cu — HLL.Compute on the device: the distinct-count estimate of every group of an AGGR_HLL state, bit for
// bit what the reference computes on the host from the same register vectors (query/common/hll.go:735-775; restated in
// aresdb_b200/postprocess.py hll_estimate, which the tests compare against).
//
// Input: the register vectors of AggStateFinalizeHLL (per group either count x 4 bytes (rho+1) << 16 | reg, count <
// HLL_DENSE_THRESHOLD, in ascending register order, or HLL_DENSE_SIZE bytes of rho+1) and the u16 register counts.
//
// The sum of 2^-v (v = rho+1, 0 for an empty register of a dense vector) decides the last bits of the raw estimate, and
// the reference adds it in float64 in vector order.  When every v of a group is <= 39, every partial sum is a multiple of
// 2^-39 no larger than 2^14, which 53 bits hold: each of those additions is exact, so the ordered sum IS the exact sum,
// and one CTA accumulates it in any order as an integer in units of 2^-39.  A group holding some v >= 40 (a register hit
// with probability ~2^-38 per row) is walked by one thread in the reference's order instead.
//
// The rest is the reference's scalar code with explicitly rounded operations (no FMA contraction), its bias table
// (__constant__ below), and a host-built table of m * log(m / (m - nonzero)) for linear counting: the host's log (glibc's,
// the one Python's math.log calls) rather than CUDA's log, which is not correctly rounded.
#include <cmath>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace aresb {

namespace {

constexpr int kEstThreads = 256;
constexpr int kUnitBits = 39;                     // the integer sum counts units of 2^-39
constexpr int kBiasK = 6;                         // getEstimateBias: mean bias of the 6 nearest raw estimates
constexpr int kBiasEntries = 201;
constexpr double kM = (double)HLL_DENSE_SIZE;     // m = 2^14 registers
constexpr double kThreshold = 15500.0;            // HLL_THRESHOLD of p = 14

// HyperLogLog++ empirical bias data for p = 14 (Heule, Nunkesser, Hall, "HyperLogLog in Practice", Google 2013,
// appendix): raw estimate -> measured bias.  Same data as aresdb_b200/hll_bias_p14.py.
__constant__ double cRawEstimates[kBiasEntries] = {
    11817.475, 12015.0046, 12215.3792, 12417.7504, 12623.1814, 12830.0086, 13040.0072, 13252.503, 13466.178, 13683.2738,
    13902.0344, 14123.9798, 14347.394, 14573.7784, 14802.6894, 15033.6824, 15266.9134, 15502.8624, 15741.4944,
    15980.7956, 16223.8916, 16468.6316, 16715.733, 16965.5726, 17217.204, 17470.666, 17727.8516, 17986.7886, 18247.6902,
    18510.9632, 18775.304, 19044.7486, 19314.4408, 19587.202, 19862.2576, 20135.924, 20417.0324, 20697.9788, 20979.6112,
    21265.0274, 21550.723, 21841.6906, 22132.162, 22428.1406, 22722.127, 23020.5606, 23319.7394, 23620.4014, 23925.2728,
    24226.9224, 24535.581, 24845.505, 25155.9618, 25470.3828, 25785.9702, 26103.7764, 26420.4132, 26742.0186,
    27062.8852, 27388.415, 27714.6024, 28042.296, 28365.4494, 28701.1526, 29031.8008, 29364.2156, 29704.497, 30037.1458,
    30380.111, 30723.8168, 31059.5114, 31404.9498, 31751.6752, 32095.2686, 32444.7792, 32794.767, 33145.204, 33498.4226,
    33847.6502, 34209.006, 34560.849, 34919.4838, 35274.9778, 35635.1322, 35996.3266, 36359.1394, 36722.8266,
    37082.8516, 37447.7354, 37815.9606, 38191.0692, 38559.4106, 38924.8112, 39294.6726, 39663.973, 40042.261,
    40416.2036, 40779.2036, 41161.6436, 41540.9014, 41921.1998, 42294.7698, 42678.5264, 43061.3464, 43432.375,
    43818.432, 44198.6598, 44583.0138, 44970.4794, 45353.924, 45729.858, 46118.2224, 46511.5724, 46900.7386, 47280.6964,
    47668.1472, 48055.6796, 48446.9436, 48838.7146, 49217.7296, 49613.7796, 50010.7508, 50410.0208, 50793.7886,
    51190.2456, 51583.1882, 51971.0796, 52376.5338, 52763.319, 53165.5534, 53556.5594, 53948.2702, 54346.352,
    54748.7914, 55138.577, 55543.4824, 55941.1748, 56333.7746, 56745.1552, 57142.7944, 57545.2236, 57935.9956,
    58348.5268, 58737.5474, 59158.5962, 59542.6896, 59958.8004, 60349.3788, 60755.0212, 61147.6144, 61548.194,
    61946.0696, 62348.6042, 62763.603, 63162.781, 63560.635, 63974.3482, 64366.4908, 64771.5876, 65176.7346, 65597.3916,
    65995.915, 66394.0384, 66822.9396, 67203.6336, 67612.2032, 68019.0078, 68420.0388, 68821.22, 69235.8388, 69640.0724,
    70055.155, 70466.357, 70863.4266, 71276.2482, 71677.0306, 72080.2006, 72493.0214, 72893.5952, 73314.5856,
    73714.9852, 74125.3022, 74521.2122, 74933.6814, 75341.5904, 75743.0244, 76166.0278, 76572.1322, 76973.1028,
    77381.6284, 77800.6092, 78189.328, 78607.0962, 79012.2508, 79407.8358, 79825.725, 80238.701, 80646.891, 81035.6436,
    81460.0448, 81876.3884,
};
__constant__ double cBiases[kBiasEntries] = {
    11816.475, 11605.0046, 11395.3792, 11188.7504, 10984.1814, 10782.0086, 10582.0072, 10384.503, 10189.178, 9996.2738,
    9806.0344, 9617.9798, 9431.394, 9248.7784, 9067.6894, 8889.6824, 8712.9134, 8538.8624, 8368.4944, 8197.7956,
    8031.8916, 7866.6316, 7703.733, 7544.5726, 7386.204, 7230.666, 7077.8516, 6926.7886, 6778.6902, 6631.9632, 6487.304,
    6346.7486, 6206.4408, 6070.202, 5935.2576, 5799.924, 5671.0324, 5541.9788, 5414.6112, 5290.0274, 5166.723,
    5047.6906, 4929.162, 4815.1406, 4699.127, 4588.5606, 4477.7394, 4369.4014, 4264.2728, 4155.9224, 4055.581, 3955.505,
    3856.9618, 3761.3828, 3666.9702, 3575.7764, 3482.4132, 3395.0186, 3305.8852, 3221.415, 3138.6024, 3056.296,
    2970.4494, 2896.1526, 2816.8008, 2740.2156, 2670.497, 2594.1458, 2527.111, 2460.8168, 2387.5114, 2322.9498,
    2260.6752, 2194.2686, 2133.7792, 2074.767, 2015.204, 1959.4226, 1898.6502, 1850.006, 1792.849, 1741.4838, 1687.9778,
    1638.1322, 1589.3266, 1543.1394, 1496.8266, 1447.8516, 1402.7354, 1361.9606, 1327.0692, 1285.4106, 1241.8112,
    1201.6726, 1161.973, 1130.261, 1094.2036, 1048.2036, 1020.6436, 990.901400000002, 961.199800000002,
    924.769800000002, 899.526400000002, 872.346400000002, 834.375, 810.432000000001, 780.659800000001, 756.013800000001,
    733.479399999997, 707.923999999999, 673.858, 652.222399999999, 636.572399999997, 615.738599999997, 586.696400000001,
    564.147199999999, 541.679600000003, 523.943599999999, 505.714599999999, 475.729599999999, 461.779600000002,
    449.750800000002, 439.020799999998, 412.7886, 400.245600000002, 383.188199999997, 362.079599999997,
    357.533799999997, 334.319000000003, 327.553399999997, 308.559399999998, 291.270199999999, 279.351999999999,
    271.791400000002, 252.576999999997, 247.482400000001, 236.174800000001, 218.774599999997, 220.155200000001,
    208.794399999999, 201.223599999998, 182.995600000002, 185.5268, 164.547400000003, 176.5962, 150.689599999998,
    157.8004, 138.378799999999, 134.021200000003, 117.614399999999, 108.194000000003, 97.0696000000025,
    89.6042000000016, 95.6030000000028, 84.7810000000027, 72.635000000002, 77.3482000000004, 59.4907999999996,
    55.5875999999989, 50.7346000000034, 61.3916000000027, 50.9149999999936, 39.0384000000049, 58.9395999999979,
    29.633600000001, 28.2032000000036, 26.0078000000067, 17.0387999999948, 9.22000000000116, 13.8387999999977,
    8.07240000000456, 14.1549999999988, 15.3570000000036, 3.42660000000615, 6.24820000000182, -2.96940000000177,
    -8.79940000000352, -5.97860000000219, -14.4048000000039, -3.4143999999942, -13.0148000000045, -11.6977999999945,
    -25.7878000000055, -22.3185999999987, -24.409599999999, -31.9756000000052, -18.9722000000038, -22.8678000000073,
    -30.8972000000067, -32.3715999999986, -22.3907999999938, -43.6720000000059, -35.9038, -39.7492000000057,
    -54.1641999999993, -45.2749999999942, -42.2989999999991, -44.1089999999967, -64.3564000000042, -49.9551999999967,
    -42.6116000000038,
};

// 2^-v, exactly (what the reference's 1.0 / float64(1 << v) is), for v in 0..1022
__device__ __forceinline__ double pow2Neg(uint32_t v) { return __longlong_as_double((long long)(1023 - (int)v) << 52); }

// 2^-v in units of 2^-39, v <= 39
__device__ __forceinline__ unsigned long long unitsOf(uint32_t v) { return v <= kUnitBits ? 1ull << (kUnitBits - v) : 0ull; }

// getEstimateBias (query/common/hll.go:639-667): the insertion point i of `e` (bisect right), the window
// [max(i - 1 - k, 0), min(i + k, n)), its k entries nearest to e in (squared distance, index) order, and the mean of their
// biases summed in that order.  The window (at most 2k + 1 entries) is held in registers: every index into it is a
// compile-time constant.
__device__ double estimateBias(double e) {
  int lo = 0, hi = kBiasEntries;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (e < cRawEstimates[mid]) hi = mid; else lo = mid + 1;
  }
  const int first = max(lo - 1 - kBiasK, 0), end = min(lo + kBiasK, kBiasEntries);
  double dist[2 * kBiasK + 1];
  uint32_t taken = 0;
#pragma unroll
  for (int w = 0; w < 2 * kBiasK + 1; w++) {
    const double d = first + w < end ? __dsub_rn(cRawEstimates[first + w], e) : 0.0;
    dist[w] = __dmul_rn(d, d);
    if (first + w >= end) taken |= 1u << w;
  }
  double sum = 0.0;
  for (int r = 0; r < kBiasK; r++) {
    int best = -1;
    double bestD = 0.0;
#pragma unroll
    for (int w = 0; w < 2 * kBiasK + 1; w++)   // ascending w: the smaller index wins a tie
      if (!(taken >> w & 1u) && (best < 0 || dist[w] < bestD)) { best = w; bestD = dist[w]; }
    taken |= 1u << best;
    sum = __dadd_rn(sum, cBiases[first + best]);
  }
  return __ddiv_rn(sum, (double)kBiasK);
}

// Byte offset of every group's vector: exclusive prefix of its size (the sizing rule of the vectors' producers), one CTA.
__global__ void __launch_bounds__(1024)
hllVectorOffsetsKernel(const uint16_t *__restrict__ counts, int n, unsigned long long *__restrict__ offsets) {
  __shared__ unsigned long long sWarp[32];
  __shared__ unsigned long long sCarry;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) sCarry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t c = i < n ? counts[i] : 0u;
    const unsigned long long x = c < (uint32_t)HLL_DENSE_THRESHOLD ? 4ull * c : (unsigned long long)HLL_DENSE_SIZE;
    unsigned long long inc = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, inc, d);
      if (lane >= (uint32_t)d) inc += y;
    }
    if (lane == 31) sWarp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      const unsigned long long v = sWarp[lane];
      unsigned long long s = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, s, d);
        if (lane >= (uint32_t)d) s += y;
      }
      sWarp[lane] = s - v;
    }
    __syncthreads();
    if (i < n) offsets[i] = sCarry + sWarp[warp] + inc - x;
    __syncthreads();
    if (threadIdx.x == 1023) sCarry += sWarp[31] + inc;   // (the last thread's inclusive prefix is the tile's total)
    __syncthreads();
  }
}

// One CTA per group: the sum of 2^-v as an integer (or, with some v >= 40, in the reference's order by one thread),
// the number of hit registers, then HLL.Compute's scalar steps.
__global__ void __launch_bounds__(kEstThreads)
hllEstimateKernel(const uint8_t *__restrict__ vec, const uint16_t *__restrict__ counts, const unsigned long long *__restrict__ offsets,
                  const double *__restrict__ linearCounting, double *__restrict__ out) {
  __shared__ unsigned long long sUnits[kEstThreads / 32];
  __shared__ uint32_t sNonzero[kEstThreads / 32], sMax[kEstThreads / 32];
  const uint32_t g = blockIdx.x, c = counts[g];
  const bool sparse = c < (uint32_t)HLL_DENSE_THRESHOLD;
  // every vector starts at a multiple of 4 bytes
  const uint32_t *words = reinterpret_cast<const uint32_t *>(vec + offsets[g]);
  unsigned long long units = 0;
  uint32_t nonzero = 0, maxV = 0;
  if (sparse) {
    for (uint32_t k = threadIdx.x; k < c; k += kEstThreads) {
      const uint32_t v = words[k] >> 16;
      units += unitsOf(v);
      maxV = max(maxV, v);
    }
    nonzero = threadIdx.x == 0 ? c : 0u;
  } else {
    for (uint32_t k = threadIdx.x; k < (uint32_t)HLL_DENSE_SIZE / 4; k += kEstThreads) {
      const uint32_t w = words[k];
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const uint32_t v = (w >> (8 * b)) & 0xFFu;
        units += unitsOf(v);
        nonzero += v != 0;
        maxV = max(maxV, v);
      }
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    units += __shfl_down_sync(0xFFFFFFFFu, units, d);
    nonzero += __shfl_down_sync(0xFFFFFFFFu, nonzero, d);
    maxV = max(maxV, __shfl_down_sync(0xFFFFFFFFu, maxV, d));
  }
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { sUnits[warp] = units; sNonzero[warp] = nonzero; sMax[warp] = maxV; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < kEstThreads / 32; w++) { units += sUnits[w]; nonzero += sNonzero[w]; maxV = max(maxV, sMax[w]); }

  double s;
  if (maxV <= (uint32_t)kUnitBits) {
    // the empty registers add 2^0 each: in the dense walk (v = 0), or as m - nonzero after the sparse entries
    if (sparse) units += (unsigned long long)(HLL_DENSE_SIZE - nonzero) << kUnitBits;
    s = __dmul_rn(__ull2double_rn(units), 0x1p-39);   // units <= 2^53: both steps exact
  } else {
    s = 0.0;
    if (sparse) {
      for (uint32_t k = 0; k < c; k++) s = __dadd_rn(s, pow2Neg(words[k] >> 16));
      s = __dadd_rn(s, __dsub_rn(kM, (double)nonzero));
    } else {
      const uint8_t *bytes = reinterpret_cast<const uint8_t *>(words);
      for (uint32_t k = 0; k < (uint32_t)HLL_DENSE_SIZE; k++) s = __dadd_rn(s, pow2Neg(bytes[k]));
    }
  }
  // 0.7213 / (1 + 1.079 / m) * m * m / s, left to right, each step rounded once
  const double alphaMM = __dmul_rn(__dmul_rn(__ddiv_rn(0.7213, __dadd_rn(1.0, __ddiv_rn(1.079, kM))), kM), kM);
  double estimate = __ddiv_rn(alphaMM, s);
  if (estimate <= 5.0 * kM) estimate = __dsub_rn(estimate, estimateBias(estimate));
  double linear = estimate;
  if (nonzero < (uint32_t)HLL_DENSE_SIZE) linear = linearCounting[nonzero];
  if (linear <= kThreshold) estimate = linear;
  out[g] = trunc(estimate);
}

constexpr int kMaxDevices = 64;

// m * log(m / (m - n)) for n = 0..m-1 in the reference's expression, computed once per device with the host's log
// (glibc's, which Python's math.log calls too) and kept for the life of the process.
const double *linearCountingTable() {
  static std::mutex mu;
  static double *tables[kMaxDevices] = {};
  int dev = 0;
  ARES_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices) throw EngineError("device ordinal out of range");
  std::lock_guard<std::mutex> lock(mu);
  if (tables[dev] == nullptr) {
    std::vector<double> host(HLL_DENSE_SIZE);
    for (int n = 0; n < HLL_DENSE_SIZE; n++) host[n] = kM * std::log(kM / (kM - n));
    void *p = nullptr;
    ARES_CUDA(cudaMalloc(&p, sizeof(double) * host.size()));
    ARES_CUDA(cudaMemcpy(p, host.data(), sizeof(double) * host.size(), cudaMemcpyHostToDevice));
    tables[dev] = static_cast<double *>(p);
  }
  return tables[dev];
}

}  // namespace

// The estimates of `groups` register vectors (AggStateFinalizeHLL's layout) into out[0..groups).  Asynchronous.
void hllEstimates(const uint8_t *vec, const uint16_t *counts, int groups, double *out, cudaStream_t s) {
  const double *linear = linearCountingTable();
  Scratch offsets(sizeof(unsigned long long) * (size_t)groups, s);
  hllVectorOffsetsKernel<<<1, 1024, 0, s>>>(counts, groups, offsets.as<unsigned long long>());
  checkLastError("hllVectorOffsets");
  hllEstimateKernel<<<groups, kEstThreads, 0, s>>>(vec, counts, offsets.as<unsigned long long>(), linear, out);
  checkLastError("hllEstimate");
}

}  // namespace aresb

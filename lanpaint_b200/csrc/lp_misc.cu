// lanpaint_b200: library plumbing (options, status, per-device facts, geometry) and the small utility kernels.
#include "lp_common.cuh"

namespace lp {

thread_local int g_last_cuda_error = 0;

// process-wide switches, initialised from the environment, adjustable through lp_set_option()
int g_opt_pdl = [] {
  const char* e = getenv("LANPAINT_B200_PDL");
  return (e && e[0] == '0') ? 0 : 1;
}();
int g_opt_tma = [] {
  const char* e = getenv("LANPAINT_B200_TMA");
  return e ? atoi(e) : 1;
}();
int g_opt_tma_min = [] {
  const char* e = getenv("LANPAINT_B200_TMA_MIN");
  return e ? atoi(e) : (1 << 18);
}();

// Inside a job the LDG boundary kernel's inputs were just written by the network and sit in L2, and it skips the
// operands a vector's mask makes unnecessary, so it is the default; the TMA-staged variant stays available, off.
int g_opt_tma_boundary = [] {
  const char* e = getenv("LANPAINT_B200_TMA_BOUNDARY");
  return e ? atoi(e) : 0;
}();
int g_opt_l2_handoff = [] {
  const char* e = getenv("LANPAINT_B200_L2_HANDOFF");
  return e ? atoi(e) : kL2Default;
}();
int g_opt_discard_heads = 1;

int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}

const DeviceInfo& device_info(int device) {
  static DeviceInfo info[kMaxDevices] = {};
  static DeviceInfo fallback = {132, 2048};  // H100 SXM
  if (device < 0 || device >= kMaxDevices) return fallback;
  DeviceInfo& d = info[device];
  if (d.sms == 0) {  // benign race: every thread writes the same values
    int sms = 0, tpsm = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
        cudaDeviceGetAttribute(&tpsm, cudaDevAttrMaxThreadsPerMultiProcessor, device) != cudaSuccess) {
      g_last_cuda_error = static_cast<int>(cudaGetLastError());
      return fallback;
    }
    d.threads_per_sm = tpsm;
    d.sms = sms;
  }
  return d;
}

// Exact for every n < 2^31: with l = ceil(log2 d), mul = floor(2^(31+l)/d) + 1 < 2^32 and the error
// n * eps / 2^(31+l) stays below 1/d.  d == 1 is flagged with mul == 0.
FastDiv make_fastdiv(uint32_t d) {
  FastDiv f{d, 0u, 0u};
  if (d <= 1) return f;
  uint32_t l = 0;
  while ((1ull << l) < d) ++l;
  const unsigned shift = 31 + l;
  f.mul = static_cast<uint32_t>(((1ull << shift) / d) + 1);
  f.shift = l - 1;
  return f;
}

int make_geometry(const lp_dims* d, Geometry& g) {
  if (!d || d->n_rows < 0 || d->per_row <= 0 || d->spatial <= 0) return LP_ERR_INVALID;
  if (d->per_row % d->spatial != 0) return LP_ERR_INVALID;
  if (d->mask_row_stride < 0 || d->mask_channel_stride < 0) return LP_ERR_INVALID;
  const int64_t total = d->n_rows * d->per_row;
  const int64_t mask_extent = d->n_rows * d->mask_row_stride + d->per_row;  // loose upper bound
  if (total >= (int64_t(1) << 31) || mask_extent >= (int64_t(1) << 31)) return LP_ERR_UNSUPPORTED;
  g.total = static_cast<uint32_t>(total);
  g.per_row = make_fastdiv(static_cast<uint32_t>(d->per_row));
  g.spatial = make_fastdiv(static_cast<uint32_t>(d->spatial));
  g.mask_row_stride = static_cast<uint32_t>(d->mask_row_stride);
  g.mask_channel_stride = static_cast<uint32_t>(d->mask_channel_stride);
  if (d->row_split < 0 || d->row_split > d->per_row) return LP_ERR_INVALID;
  g.n_rows = static_cast<uint32_t>(d->n_rows);
  g.row_split = static_cast<uint32_t>(d->row_split);
  return LP_OK;
}

// Geometry of torch's own randn kernel (ATen/native/cuda/DistributionTemplates.h: calc_execution_policy).
int torch_grid(int64_t numel, int device, int64_t* grid, uint64_t* inc) {
  if (numel <= 0) return LP_ERR_INVALID;
  if (device < 0) device = current_device();
  if (device < 0) return LP_ERR_CUDA;
  const DeviceInfo& d = device_info(device);
  int64_t g = (numel + 255) / 256;
  const int64_t cap = int64_t(d.sms) * (d.threads_per_sm / 256);
  if (g > cap) g = cap;
  if (grid) *grid = g;
  if (inc) *inc = (uint64_t)(((numel - 1) / (256 * g * 4) + 1) * 4);
  return LP_OK;
}

__global__ void __launch_bounds__(kBlock) pack_mask_kernel(const float* __restrict__ m, uint8_t* out,
                                                           uint32_t n, int invert) {
  pdl_prologue();
  const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const bool hi = __ldg(m + i) > 0.5f;
  out[i] = (hi != (invert != 0)) ? 1 : 0;
}

// ---- the known-operand layout (lp_known): three launches, once per job -------------------------------------
// Words are handled in blocks of kBlock; words[2W..2W+1] is the end sentinel {0, known count}, and the tail of the
// buffer holds one count per block of words for the scan.
inline uint32_t known_word_count(uint32_t total) { return (total + 31u) / 32u + 1u; }  // W + the sentinel

// Inclusive prefix sum over the kBlock threads of a block (Hillis-Steele in shared memory).
__device__ __forceinline__ uint32_t block_inclusive_sum(uint32_t v, uint32_t* s) {
  s[threadIdx.x] = v;
  __syncthreads();
#pragma unroll
  for (int o = 1; o < kBlock; o <<= 1) {
    const uint32_t add = threadIdx.x >= (uint32_t)o ? s[threadIdx.x - o] : 0u;
    __syncthreads();
    s[threadIdx.x] += add;
    __syncthreads();
  }
  return s[threadIdx.x];
}

// words[2w] = known bits of elements 32w..32w+31 (through the mask's strides); block_sums[b] = known elements of
// word block b
__global__ void __launch_bounds__(kBlock) known_bits_kernel(const uint8_t* __restrict__ mask, Geometry g,
                                                            uint32_t* words, uint32_t* block_sums, uint32_t n_words) {
  __shared__ uint32_t s[kBlock];
  pdl_prologue();
  const uint32_t w = blockIdx.x * kBlock + threadIdx.x;
  uint32_t bits = 0;
  if (w < n_words) {
    for (uint32_t b = 0; b < 32u; ++b) {
      const uint32_t e = 32u * w + b;
      if (e >= g.total) break;
      uint32_t row, mi;
      locate(g, e, row, mi);
      bits |= (__ldg(mask + mi) != 0 ? 1u : 0u) << b;
    }
    words[2u * w] = bits;
  }
  const uint32_t sum = block_inclusive_sum(__popc(bits), s);
  if (threadIdx.x == kBlock - 1) block_sums[blockIdx.x] = sum;
}

// block_sums -> their exclusive prefix sums, in place (one CTA)
__global__ void __launch_bounds__(kBlock) known_scan_kernel(uint32_t* block_sums, uint32_t n_blocks) {
  __shared__ uint32_t s[kBlock];
  pdl_prologue();
  uint32_t carry = 0;
  for (uint32_t base = 0; base < n_blocks; base += kBlock) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < n_blocks ? block_sums[i] : 0u;
    const uint32_t inc = block_inclusive_sum(v, s);
    if (i < n_blocks) block_sums[i] = carry + inc - v;
    carry += s[kBlock - 1];
    __syncthreads();
  }
}

// words[2w + 1] = known elements before 32w; then every known element's y (and noise) to its packed index
__global__ void __launch_bounds__(kBlock) known_scatter_kernel(uint32_t* words, const uint32_t* __restrict__ block_sums,
                                                               uint32_t n_words, uint32_t total,
                                                               const float* __restrict__ y,
                                                               const float* __restrict__ noise, float* yk, float* nk) {
  __shared__ uint32_t s[kBlock], sbits[kBlock], sbase[kBlock];
  pdl_prologue();
  const uint32_t w = blockIdx.x * kBlock + threadIdx.x;
  const uint32_t bits = w < n_words ? words[2u * w] : 0u;
  const uint32_t c = __popc(bits);
  const uint32_t base = block_sums[blockIdx.x] + block_inclusive_sum(c, s) - c;
  if (w < n_words) words[2u * w + 1u] = base;
  sbits[threadIdx.x] = bits;
  sbase[threadIdx.x] = base;
  __syncthreads();
  const uint32_t e0 = blockIdx.x * kBlock * 32u;
  const uint32_t e1 = e0 >= total ? e0 : (total - e0 < kBlock * 32u ? total : e0 + kBlock * 32u);
  for (uint32_t e = e0 + threadIdx.x; e < e1; e += kBlock) {
    const uint32_t wl = (e - e0) >> 5, b = e & 31u;
    const uint32_t m = sbits[wl];
    if ((m >> b) & 1u) {
      const uint32_t idx = sbase[wl] + __popc(m & ((1u << b) - 1u));
      yk[idx] = __ldg(y + e);
      if (nk) nk[idx] = __ldg(noise + e);
    }
  }
}

__global__ void __launch_bounds__(kBlock) fill_normal_philox_kernel(float* out, uint32_t n, uint64_t seed,
                                                                    uint64_t draw, const uint64_t* st) {
  pdl_prologue();
  const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  if (st) {
    seed = st[0];
    draw += st[1];
  }
  out[i] = pick(philox_normal4(seed, draw, i >> 2), i & 3);
}

__global__ void __launch_bounds__(kBlock) fill_normal_torch_kernel(float* out, uint32_t n, uint64_t seed,
                                                                   uint64_t offset, const uint64_t* st,
                                                                   uint32_t T) {
  pdl_prologue();
  const uint32_t tid = blockIdx.x * kBlock + threadIdx.x;
  if (tid >= T) return;
  if (st) {
    seed = st[0];
    offset += st[1];
  }
  uint32_t call = 0;
  for (uint64_t base = tid; base < n; base += 4ull * T, ++call) {
    const float4 r = torch_normal4(seed, offset, tid, call);
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const uint64_t li = base + (uint64_t)ii * T;
      if (li < n) out[li] = pick(r, ii);
    }
  }
}

// bitwise comparison of the lane-pair Box-Muller with the scalar cuRAND form over pseudo-random and edge-case inputs
__global__ void __launch_bounds__(kBlock) selftest_box_muller_kernel(uint64_t n, uint64_t seed, unsigned long long* bad) {
  const uint64_t gid = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * kBlock;
  unsigned long long mine = 0;
  for (uint64_t i = gid; i < n; i += stride) {
    uint4 r = philox4x32_10(make_uint4((uint32_t)i, (uint32_t)(i >> 32), 0x5eedu, 0u),
                            make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    if (i < 4096) {  // edge cases: the extremes of u and v in every combination, u == 1 (log = 0), smallest u
      const uint32_t edge[8] = {0u, 1u, 0x7fffffffu, 0x80000000u, 0xffffff00u, 0xffffff7fu, 0xffffff80u, 0xffffffffu};
      r.x = edge[i & 7];
      r.y = edge[(i >> 3) & 7];
      r.z = edge[(i >> 6) & 7];
      r.w = edge[(i >> 9) & 7];
    }
    const float2 a = box_muller_curand(r.x, r.y), b = box_muller_curand(r.z, r.w);
    float2 c, d;
    box_muller_curand_x2(r.x, r.y, r.z, r.w, c, d);
    mine += (__float_as_uint(a.x) != __float_as_uint(c.x)) + (__float_as_uint(a.y) != __float_as_uint(c.y)) +
            (__float_as_uint(b.x) != __float_as_uint(d.x)) + (__float_as_uint(b.y) != __float_as_uint(d.y));
  }
  if (mine) atomicAdd(bad, mine);
}

// box_muller_fast (the LP_RNG_PHILOX transform) over all 2^32 values of one input word, the other word fixed:
// counts non-finite outputs and takes the largest |fast - fp64 Box-Muller of the same fp32 u and v|
__global__ void __launch_bounds__(kBlock) selftest_normal_fast_kernel(uint32_t fixed, int sweep_second,
                                                                      unsigned long long* nonfinite,
                                                                      unsigned long long* max_err_bits) {
  pdl_prologue();
  const uint64_t gid = (uint64_t)blockIdx.x * kBlock + threadIdx.x;
  const uint64_t stride = (uint64_t)gridDim.x * kBlock;
  unsigned long long bad = 0;
  double worst = 0.0;
  for (uint64_t w = gid; w < (1ull << 32); w += stride) {
    const uint32_t a = sweep_second ? fixed : (uint32_t)w, b = sweep_second ? (uint32_t)w : fixed;
    const float2 r = box_muller_fast(a, b);
    if (!isfinite(r.x) || !isfinite(r.y)) {
      ++bad;
      continue;
    }
    // the fp32 u and v box_muller_fast starts from, then the transform in fp64
    const float u = a * 2.3283064e-10f + (2.3283064e-10f / 2);
    const float v = b * (2.3283064e-10f * 6.2831855f) + ((2.3283064e-10f * 6.2831855f) / 2);
    const double s = sqrt(-2.0 * log((double)u));
    double sn, cs;
    sincos((double)v, &sn, &cs);
    worst = fmax(worst, fmax(fabs((double)r.x - s * sn), fabs((double)r.y - s * cs)));
  }
  for (int o = 16; o > 0; o >>= 1) {
    bad += __shfl_xor_sync(0xffffffffu, bad, o);
    worst = fmax(worst, __shfl_xor_sync(0xffffffffu, worst, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (bad) atomicAdd(nonfinite, bad);
    atomicMax(max_err_bits, (unsigned long long)__double_as_longlong(worst));  // worst >= 0: bits order like values
  }
}

template <int N, typename H>
__global__ void __launch_bounds__(kBlock) synth_denoiser_kernel(const float* __restrict__ x, H* h0, H* h1, uint32_t n,
                                                                float a0, float b0, float c0, float a1, float c1) {
  pdl_prologue();
  const uint32_t i = (blockIdx.x * kBlock + threadIdx.x) * N;
  if (i >= n) return;
  float xv[N], u[N], w[N];
  load_f_ro<N>(x, i, xv);
#pragma unroll
  for (int j = 0; j < N; ++j) {
    u[j] = fmaf(a0, xv[j], fmaf(b0, tanhf(xv[j]), c0));
    w[j] = fmaf(a1, xv[j], c1);
  }
  if constexpr (sizeof(H) == 4) {
    store_f<N>(reinterpret_cast<float*>(h0), i, u);
    if (h1) store_f<N>(reinterpret_cast<float*>(h1), i, w);
  } else {
#pragma unroll
    for (int j = 0; j < N; ++j) {   // narrow stores of N consecutive 16-bit values
      if constexpr (sizeof(H) == 2) {
        h0[i + j] = H(u[j]);
        if (h1) h1[i + j] = H(w[j]);
      }
    }
  }
}

template <typename H>
int launch_synth(const float* x, void* h0, void* h1, int64_t n, const float* coef, cudaStream_t s) {
  const bool v4 = n % 4 == 0 && aligned16(x) && aligned16(h0) && (!h1 || aligned16(h1));
  if (v4)
    launch_kernel(synth_denoiser_kernel<4, H>, dim3(blocks_for((uint32_t)n / 4)), s, x, static_cast<H*>(h0),
                  static_cast<H*>(h1), (uint32_t)n, coef[0], coef[1], coef[2], coef[3], coef[4]);
  else
    launch_kernel(synth_denoiser_kernel<1, H>, dim3(blocks_for((uint32_t)n)), s, x, static_cast<H*>(h0),
                  static_cast<H*>(h1), (uint32_t)n, coef[0], coef[1], coef[2], coef[3], coef[4]);
  return check_launch();
}

}  // namespace lp

// ============================================================================
// C ABI
// ============================================================================
using namespace lp;

extern "C" int lp_abi_version(void) { return LP_ABI_VERSION; }

extern "C" const char* lp_status_string(int status) {
  switch (status) {
    case LP_OK: return "ok";
    case LP_ERR_INVALID: return "invalid argument";
    case LP_ERR_ALIGNMENT: return "misaligned pointer";
    case LP_ERR_CUDA: return "CUDA launch failed (see lp_last_cuda_error)";
    case LP_ERR_UNSUPPORTED: return "unsupported size (>= 2^31 elements)";
    default: return "unknown status";
  }
}

extern "C" int lp_last_cuda_error(void) { return g_last_cuda_error; }

extern "C" int lp_set_option(const char* name, int value) {
  if (!name) return LP_ERR_INVALID;
  const auto eq = [&](const char* k) { int i = 0; while (k[i] && name[i] == k[i]) ++i; return !k[i] && !name[i]; };
  if (eq("pdl")) { g_opt_pdl = value; return LP_OK; }
  if (eq("tma")) { g_opt_tma = value; return LP_OK; }
  if (eq("tma_min")) { g_opt_tma_min = value; return LP_OK; }
  if (eq("tma_boundary")) { g_opt_tma_boundary = value; return LP_OK; }
  if (eq("l2_handoff")) { g_opt_l2_handoff = value; return LP_OK; }
  if (eq("discard_heads")) { g_opt_discard_heads = value; return LP_OK; }
  return LP_ERR_INVALID;
}

extern "C" int64_t lp_selftest_index_math(int64_t samples) {
  int64_t bad = 0;
  auto check = [&](uint32_t n, uint32_t d) {
    const FastDiv f = make_fastdiv(d);
    const uint32_t q = f.mul ? (uint32_t)((((uint64_t)n * f.mul) >> 32) >> f.shift) : n;  // == FastDiv::div
    if (q != n / d) ++bad;
  };
  const uint32_t ds[] = {1u, 2u, 3u, 4u, 5u, 7u, 35u, 105u, 1024u, 3600u, 16384u, 65536u, 75600u, 1209600u,
                         (1u << 30), (1u << 31) - 1u, 0x7fffffffu, 1000003u};
  const uint32_t ns[] = {0u, 1u, 2u, 3u, 1023u, 65535u, 65536u, (1u << 31) - 1u, (1u << 31) - 2u, 0x40000000u};
  for (uint32_t d : ds)
    for (uint32_t n : ns) {
      check(n, d);
      if (d > 1 && n >= d) { check(n - n % d, d); check(n - n % d - 1, d); }
    }
  uint64_t st = 0x9E3779B97F4A7C15ull;
  for (int64_t k = 0; k < samples; ++k) {
    st = st * 6364136223846793005ull + 1442695040888963407ull;
    const uint32_t n = (uint32_t)(st >> 33);                       // < 2^31
    st = st * 6364136223846793005ull + 1442695040888963407ull;
    uint32_t d = (uint32_t)(st >> 33) >> ((st >> 20) & 31);        // all magnitudes
    if (d == 0) d = 1;
    check(n, d);
  }
  return bad;
}

extern "C" int lp_selftest_box_muller(int64_t n, uint64_t seed, unsigned long long* mismatches_dev, lp_stream_t stream) {
  if (n < 0 || !mismatches_dev) return LP_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(mismatches_dev, 0, sizeof(unsigned long long), s) != cudaSuccess) return (check_launch(), LP_ERR_CUDA);
  if (n == 0) return LP_OK;
  const unsigned grid = (unsigned)device_info(current_device()).sms * 8u;
  launch_kernel(selftest_box_muller_kernel, dim3(grid), s, (uint64_t)n, seed, mismatches_dev);
  return check_launch();
}

extern "C" int lp_selftest_normal_fast(uint32_t fixed_word, int sweep_second, unsigned long long* nonfinite_dev,
                                       double* max_err_dev, lp_stream_t stream) {
  if (!nonfinite_dev || !max_err_dev) return LP_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemsetAsync(nonfinite_dev, 0, sizeof(unsigned long long), s) != cudaSuccess ||
      cudaMemsetAsync(max_err_dev, 0, sizeof(double), s) != cudaSuccess)
    return (check_launch(), LP_ERR_CUDA);
  const unsigned grid = (unsigned)device_info(current_device()).sms * 8u;
  launch_kernel(selftest_normal_fast_kernel, dim3(grid), s, fixed_word, sweep_second, nonfinite_dev,
                reinterpret_cast<unsigned long long*>(max_err_dev));
  return check_launch();
}

extern "C" int lp_torch_randn_geometry(int64_t numel, int device, int64_t* grid_out, uint64_t* increment_out) {
  return torch_grid(numel, device, grid_out, increment_out);
}

extern "C" int lp_pack_mask_f32(const float* mask_f32, uint8_t* mask_u8, int64_t n, int invert,
                                lp_stream_t stream) {
  if (!mask_f32 || !mask_u8 || n < 0) return LP_ERR_INVALID;
  if (n >= (int64_t(1) << 31)) return LP_ERR_UNSUPPORTED;
  if (n == 0) return LP_OK;
  launch_kernel(pack_mask_kernel, dim3(blocks_for((uint32_t)n)), (cudaStream_t)stream, mask_f32, mask_u8,
                                                                                 (uint32_t)n, invert);
  return check_launch();
}

extern "C" int64_t lp_known_words(int64_t total) {
  if (total < 0 || total >= (int64_t(1) << 31)) return -1;
  const int64_t n_words = known_word_count((uint32_t)total);
  return 2 * n_words + (n_words + kBlock - 1) / kBlock;
}

extern "C" int lp_pack_known(const uint8_t* mask, const lp_dims* dims, const float* y, const float* noise,
                             uint32_t* words, float* y_known, float* noise_known, lp_stream_t stream) {
  if (!mask || !y || !words || !y_known || (noise && !noise_known)) return LP_ERR_INVALID;
  Geometry g;
  if (int rc = make_geometry(dims, g)) return rc;
  const uint32_t n_words = known_word_count(g.total);
  const uint32_t n_blocks = (n_words + kBlock - 1) / kBlock;
  uint32_t* block_sums = words + 2u * n_words;
  cudaStream_t s = (cudaStream_t)stream;
  launch_kernel(known_bits_kernel, dim3(n_blocks), s, mask, g, words, block_sums, n_words);
  launch_kernel(known_scan_kernel, dim3(1), s, block_sums, n_blocks);
  launch_kernel(known_scatter_kernel, dim3(n_blocks), s, words, (const uint32_t*)block_sums, n_words, g.total, y,
                noise, y_known, noise ? noise_known : nullptr);
  return check_launch();
}

extern "C" int lp_fill_normal_f32(float* out, int64_t n, const lp_rng* rng, lp_stream_t stream) {
  if (!out || !rng || n < 0) return LP_ERR_INVALID;
  if (n >= (int64_t(1) << 31)) return LP_ERR_UNSUPPORTED;
  if (n == 0) return LP_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (rng->mode == LP_RNG_PHILOX) {
    launch_kernel(fill_normal_philox_kernel, dim3(blocks_for((uint32_t)n)), s, out, (uint32_t)n, rng->seed,
                                                                        rng->draw0, rng->state);
    return check_launch();
  }
  if (rng->mode == LP_RNG_TORCH) {
    int64_t grid = 0;
    if (int rc = torch_grid(n, -1, &grid, nullptr)) return rc;
    launch_kernel(fill_normal_torch_kernel, dim3((unsigned)grid), s, out, (uint32_t)n, rng->seed, rng->draw0,
                                                              rng->state, (uint32_t)(grid * 256));
    return check_launch();
  }
  return LP_ERR_INVALID;
}

extern "C" int lp_synth_denoiser(const float* x, void* h0, void* h1, int dtype, int64_t n, const float* coef,
                                 lp_stream_t stream) {
  if (!x || !h0 || !coef || n < 0) return LP_ERR_INVALID;
  if (n >= (int64_t(1) << 31)) return LP_ERR_UNSUPPORTED;
  if (n == 0) return LP_OK;
  cudaStream_t s = (cudaStream_t)stream;
  switch (dtype) {
    case LP_DTYPE_F32: return launch_synth<float>(x, h0, h1, n, coef, s);
    case LP_DTYPE_BF16: return launch_synth<__nv_bfloat16>(x, h0, h1, n, coef, s);
    case LP_DTYPE_F16: return launch_synth<__half>(x, h0, h1, n, coef, s);
    default: return LP_ERR_INVALID;
  }
}

extern "C" int lp_synth_denoiser_f32(const float* x, float* h0, float* h1, int64_t n, const float* coef,
                                     lp_stream_t stream) {
  return lp_synth_denoiser(x, h0, h1, LP_DTYPE_F32, n, coef, stream);
}

extern "C" int lp_l2_persist_capacity(int device, size_t* max_persisting_bytes, size_t* max_window_bytes) {
  if (device < 0 && cudaGetDevice(&device) != cudaSuccess) return LP_ERR_CUDA;
  int a = 0, b = 0;
  if (cudaDeviceGetAttribute(&a, cudaDevAttrMaxPersistingL2CacheSize, device) != cudaSuccess ||
      cudaDeviceGetAttribute(&b, cudaDevAttrMaxAccessPolicyWindowSize, device) != cudaSuccess) {
    g_last_cuda_error = static_cast<int>(cudaGetLastError());
    return LP_ERR_CUDA;
  }
  if (max_persisting_bytes) *max_persisting_bytes = (size_t)a;
  if (max_window_bytes) *max_window_bytes = (size_t)b;
  return LP_OK;
}

extern "C" int lp_l2_persist_set(const void* ptr, size_t bytes, lp_stream_t stream) {
  if (!ptr || bytes == 0) return LP_ERR_INVALID;
  size_t cap = 0, win = 0;
  if (int rc = lp_l2_persist_capacity(-1, &cap, &win)) return rc;
  if (cap == 0 || win == 0) return LP_ERR_UNSUPPORTED;
  const size_t want = bytes < cap ? bytes : cap;
  if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) != cudaSuccess) return (check_launch(), LP_ERR_CUDA);
  cudaStreamAttrValue v;
  v.accessPolicyWindow.base_ptr = const_cast<void*>(ptr);
  v.accessPolicyWindow.num_bytes = bytes < win ? bytes : win;
  v.accessPolicyWindow.hitRatio = (float)((double)want / (double)(bytes < win ? bytes : win));
  if (v.accessPolicyWindow.hitRatio > 1.f) v.accessPolicyWindow.hitRatio = 1.f;
  v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  if (cudaStreamSetAttribute((cudaStream_t)stream, cudaStreamAttributeAccessPolicyWindow, &v) != cudaSuccess)
    return (check_launch(), LP_ERR_CUDA);
  return LP_OK;
}

extern "C" int lp_l2_persist_clear(lp_stream_t stream) {
  cudaStreamAttrValue v;
  v.accessPolicyWindow.base_ptr = nullptr;
  v.accessPolicyWindow.num_bytes = 0;
  v.accessPolicyWindow.hitRatio = 0.f;
  v.accessPolicyWindow.hitProp = cudaAccessPropertyNormal;
  v.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
  cudaStreamSetAttribute((cudaStream_t)stream, cudaStreamAttributeAccessPolicyWindow, &v);
  if (cudaCtxResetPersistingL2Cache() != cudaSuccess) return (check_launch(), LP_ERR_CUDA);
  cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0);  // give the set-aside back to normal traffic
  return LP_OK;
}

extern "C" int lp_l2_flush(void* scratch, size_t bytes, lp_stream_t stream) {
  if (!scratch) return LP_ERR_INVALID;
  if (cudaMemsetAsync(scratch, 0, bytes, (cudaStream_t)stream) != cudaSuccess) return (check_launch(), LP_ERR_CUDA);
  return LP_OK;
}

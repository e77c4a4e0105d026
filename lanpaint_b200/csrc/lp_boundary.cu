// lanpaint_b200: everything of an outer step that is not the fused sub-step.
//   prologue_kernel     replace step + change of variables              lanpaint.py:85-99
//   boundary_kernel     final paste [+ CFG combine] [+ k-diffusion Euler update] [+ next replace step]
//                       lanpaint.py:151-157, sample_euler, lanpaint.py:85-94     (LDG and TMA-staged variants)
//   boundary_ancestral_kernel / boundary_ancestral_torch_tma_kernel
//                       the same boundary for k-diffusion's sample_euler_ancestral, its randn_like drawn in-kernel
//   boundary_multistep_kernel
//                       the same boundary for k-diffusion's sample_dpmpp_2m (DPM-Solver++(2M))
//   boundary_midpoint_kernel
//                       the same boundary for either wrapper call of k-diffusion's sample_dpm_2 (DPM-Solver-2)
//   boundary_deis_kernel
//                       the same boundary for ComfyUI's sample_deis (DEIS, third order), writing the step's derivative
//   boundary_ge_kernel  the same boundary for ComfyUI's sample_gradient_estimation, writing the step's derivative
//   boundary_heun_kernel
//                       the same boundary for the second wrapper call of k-diffusion's sample_heun (its corrector)
//   advance_kernel      one un-fused advance_time_overdamped             lanpaint.py:232-254
//   stop_stats_kernel   early-stop masked reductions                     earlystop.py:32-55,238-313
#include "lp_common.cuh"

namespace lp {

// ---- prologue ----------------------------------------------------------------
template <int N>
__global__ void __launch_bounds__(kBlock) prologue_kernel(const float* x, const float* __restrict__ y,
                                                          const float* __restrict__ noise,
                                                          const uint8_t* __restrict__ mask, float* x_model,
                                                          float* x_copy, const float* __restrict__ table,
                                                          Geometry g) {
  pdl_prologue();
  const uint32_t i = (blockIdx.x * kBlock + threadIdx.x) * N;
  if (i >= g.total) return;
  uint32_t row, mi;
  locate(g, i, row, mi);
  const float rn = __ldg(table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPN);
  const float ry = __ldg(table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPY);
  float xv[N], yv[N], nv[N];
  bool known[N];
  load_f<N>(x, i, xv);
  load_f_ro<N>(y, i, yv);
  load_f_ro<N>(noise, i, nv);
  load_m<N>(mask, mi, known);
#pragma unroll
  for (int j = 0; j < N; ++j) xv[j] = known[j] ? fmaf(rn, nv[j], ry * yv[j]) : xv[j];
  store_f<N>(x_model, i, xv);
  if (x_copy) store_f<N>(x_copy, i, xv);
}

// ---- the boundary of an outer step ----------------------------------------------------
struct BoundaryArgs {
  const void* a;   // model_out (or cond)
  const void* b;   // uncond when combine
  const float* y;
  const float* noise;
  const uint8_t* mask;
  const uint32_t* kwords;  // known-operand layout (lp_known) or NULL
  const float* yk;         // y at known elements
  const float* nk;         // noise at known elements
  float* x;        // NULL: no Euler update
  float* out;      // NULL: nobody reads the denoised latent
  uint32_t out_end;  // out is stored for elements < out_end only: its first out_rows rows
  const float* next_table;  // NULL: no replace step of the next outer step
  float cfg, coef;
  int combine;
  int l2;          // kL2* bits of this launch (l2_handoff)
  int discard;     // the heads are dead after this launch (LP_HEADS_DEAD, heads_discard): the LDG boundary and the
                   // TMA-staged ancestral boundary drop their L2 lines once read
  Geometry g;
};

// per element of boundary_tma_kernel: d = combine ? b + (a-b) cfg : a ; o = known ? y : d ; x += (x - o) coef ;
// x = known ? rn n + ry y : x
__device__ __forceinline__ void boundary_element(float a, float b, float y, float nz, bool known, float& x, float& o,
                                                 bool combine, float cfg, float coef, bool euler, bool next, float rn,
                                                 float ry) {
  const float d = combine ? __fadd_rn(b, __fmul_rn(__fsub_rn(a, b), cfg)) : a;
  o = known ? y : d;
  if (euler) x = fmaf(x - o, coef, x);
  if (next) x = known ? fmaf(rn, nz, ry * y) : x;
}

// ---- the LDG boundary: one vector body, one update policy per sampler -------------------------------------------
// boundary_vector does for the N-wide vector at element i what every LDG boundary kernel shares: the known bits, y,
// the heads and the CFG combine, the pasted denoised value o = known ? y : d, the next replace step, the `out` store
// and the heads' discard.  kPk: the known bits and the packed y / noise of lp_known replace the uint8 mask and the
// dense y / noise, so y and noise cost 4 B per KNOWN element each instead of 4 B per element (a 4-wide vector is
// rarely all-free, so the dense form reads nearly all of y on a scattered mask).  The sampler's policy U supplies
//   u.load(i, update, dead)  its own operands; update: somewhere in the vector the new x is not overwritten by the
//                            replace step (any_free || !next); dead: the L2 policy of operands read for the last time
//   u.update(j, o)           element j's update from o, each operation the sampler's correctly rounded fp32 one;
//                            returns element j's new x, which the replace step then overwrites at known positions
//   u.store(i)               d_out where it has one, then x (after `out`)
//   U::kDiscard              whether the launch drops the heads' lines once read: only where a warp's vectors are
//                            one contiguous span
template <int N, typename H, bool kPk, typename U>
__device__ __forceinline__ void boundary_vector(const BoundaryArgs& p, uint32_t i, U& u) {
  const uint64_t dead = l2_policy_dead(p.l2);
  uint32_t row, mi;
  locate(p.g, i, row, mi);
  const bool next = p.next_table != nullptr;
  float av[N], bv[N], yv[N], nv[N], ov[N];
  bool known[N];
  uint32_t kb = 0, kidx = 0;
  if constexpr (kPk) {
    const uint2 w = __ldg(reinterpret_cast<const uint2*>(p.kwords) + (i >> 5));
    if constexpr (N == 4) {
      known_quad(w, i, kb, kidx);
    } else {
      kb = (w.x >> (i & 31u)) & 1u;
      kidx = w.y + __popc(w.x & ((1u << (i & 31u)) - 1u));
    }
#pragma unroll
    for (int j = 0; j < N; ++j) known[j] = ((kb >> j) & 1u) != 0;
  } else {
    load_m<N>(p.mask, mi, known);
  }
  bool any_known = false, any_free = false;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    any_known |= known[j];
    any_free |= !known[j];
  }
  const bool update = any_free || !next;
#pragma unroll
  for (int j = 0; j < N; ++j) av[j] = bv[j] = nv[j] = 0.f;
  if constexpr (kPk) {
    if constexpr (N == 4) {
      gather_known4<false>(p.yk, kb, kidx, yv);
    } else {
      yv[0] = kb ? __ldg(p.yk + kidx) : 0.f;
    }
  } else {
    load_f_ro<N>(p.y, i, yv);
  }
  // free positions: the denoised output and the running state; known positions: the re-noised clean latent
  if (any_free) {
    load_head_ro<N, H>(static_cast<const H*>(p.a), i, av, dead);
    if (p.combine) load_head_ro<N, H>(static_cast<const H*>(p.b), i, bv, dead);
  }
  u.load(i, update, dead);
  float rn = 0.f, ry = 0.f;
  if (next) {
    if constexpr (kPk) {
      if constexpr (N == 4) {
        gather_known4<false>(p.nk, kb, kidx, nv);
      } else {
        nv[0] = kb ? __ldg(p.nk + kidx) : 0.f;
      }
    } else {
      if (any_known) load_f_ro<N>(p.noise, i, nv);
    }
    rn = __ldg(p.next_table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPN);
    ry = __ldg(p.next_table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPY);
  }
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const float d = p.combine ? __fadd_rn(bv[j], __fmul_rn(__fsub_rn(av[j], bv[j]), p.cfg)) : av[j];
    const bool k = known[j];
    ov[j] = k ? yv[j] : d;
    float& x = u.update(j, ov[j]);
    if (next) x = k ? fmaf(rn, nv[j], ry * yv[j]) : x;  // rounds as prologue_kernel does
  }
  if (p.out && i < p.out_end) store_f<N>(p.out, i, ov, dead);  // a vector lies in one row
  u.store(i);
  if constexpr (U::kDiscard && 32 * N * sizeof(H) >= 128) {  // a warp's span holds whole lines
    if (p.discard) {
      const uint32_t end = i - (threadIdx.x & 31u) * N + 32u * N;  // end of this warp's span
      if (end <= p.g.total) {   // warp-uniform: a partial last warp keeps its lines
        __syncwarp();           // every lane's head loads are used
        discard_line<H>(p.a, i, end);
        if (p.b) discard_line<H>(p.b, i, end);
      }
    }
  }
}

// boundary_kernel: x += (x - o) coef, where there is an x (NULL: the paste alone)
template <int N>
struct EulerUpdate {
  static constexpr bool kDiscard = true;
  float* x;
  float coef;
  float xv[N] = {};
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t) {
    if (x && update) load_f<N>(x, i, xv);
  }
  __device__ __forceinline__ float& update(int j, float o) {
    if (x) xv[j] = fmaf(xv[j] - o, coef, xv[j]);
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) {
    if (x) store_f<N>(x, i, xv);
  }
};

template <int N, typename H, bool kPk>
__global__ void __launch_bounds__(kBlock) boundary_kernel(const BoundaryArgs p) {
  pdl_prologue();
  const uint32_t i = (walk_index(p.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
  if (i >= p.g.total) return;
  EulerUpdate<N> u{p.x, p.coef};
  boundary_vector<N, H, kPk>(p, i, u);
}

// TMA-staged persistent variant for HBM-bound sizes (fused Euler loop: x is always updated).  Same tile walk and
// mbarrier ring as substep_tma_kernel; kCombine / kNext select which slices a tile needs.
template <typename H, int kTile>
struct __align__(128) BoundaryStage {
  H a[kTile], b[kTile];
  float y[kTile], nz[kTile], x[kTile];
  uint8_t m[kTile];
};

struct BTileGeom {
  uint32_t tiles_per_channel, n_tiles, channels;
};

template <typename H, bool kCombine, bool kNext, int kTile, int kStages>
__global__ void __launch_bounds__(kBlock, 2) boundary_tma_kernel(const BoundaryArgs p, const BTileGeom tg) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  using Stage = BoundaryStage<H, kTile>;
  Stage* stage = reinterpret_cast<Stage*>(smem_raw);
  __shared__ __align__(8) uint64_t full[kStages];
  pdl_prologue();
  const uint32_t S = p.g.spatial.d;
  const H* ap = static_cast<const H*>(p.a);
  const H* bp = static_cast<const H*>(p.b);
  const uint64_t dead = l2_policy_dead(p.l2);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto tile_origin = [&](uint32_t tile, uint32_t& e0, uint32_t& len, uint32_t& row, uint32_t& mi0) {
    tile = walk_index(p.l2, tile, tg.n_tiles);  // `tile` counts in walk order
    const uint32_t rc = tile / tg.tiles_per_channel;
    const uint32_t s0 = (tile - rc * tg.tiles_per_channel) * kTile;
    len = S - s0 < (uint32_t)kTile ? S - s0 : (uint32_t)kTile;
    e0 = rc * S + s0;
    row = rc / tg.channels;
    mi0 = row * p.g.mask_row_stride + (rc - row * tg.channels) * p.g.mask_channel_stride + s0;
  };
  auto issue = [&](uint32_t tile, int s) {
    uint32_t e0, len, row, mi0;
    tile_origin(tile, e0, len, row, mi0);
    const uint32_t fb = len * 4u, hb = len * (uint32_t)sizeof(H);
    mbar_expect_tx(&full[s], fb * (2u + (kNext ? 1u : 0u)) + hb * (1u + (kCombine ? 1u : 0u)) + len);
    Stage& t = stage[s];
    tma_load_1d(t.a, ap + e0, hb, &full[s], dead);
    if (kCombine) tma_load_1d(t.b, bp + e0, hb, &full[s], dead);
    tma_load_1d(t.y, p.y + e0, fb, &full[s]);
    if (kNext) tma_load_1d(t.nz, p.noise + e0, fb, &full[s]);
    tma_load_1d(t.x, p.x + e0, fb, &full[s]);
    tma_load_1d(t.m, p.mask + mi0, len, &full[s]);
  };
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      const uint32_t tile = blockIdx.x + (uint32_t)s * gridDim.x;
      if (tile < tg.n_tiles) issue(tile, s);
    }
  }
  uint32_t k = 0;
  for (uint32_t tile = blockIdx.x; tile < tg.n_tiles; tile += gridDim.x, ++k) {
    const int s = (int)(k % kStages);
    mbar_wait(&full[s], (k / kStages) & 1u);
    uint32_t e0, len, row, mi0;
    tile_origin(tile, e0, len, row, mi0);
    const Stage& t = stage[s];
    float rn = 0.f, ry = 0.f;
    if (kNext) {
      rn = __ldg(p.next_table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPN);
      ry = __ldg(p.next_table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPY);
    }
#pragma unroll
    for (int pass = 0; pass < kTile / (4 * kBlock); ++pass) {
      const uint32_t v = threadIdx.x + pass * kBlock;
      if (4 * v < len) {
        float av[4], bv[4] = {0.f, 0.f, 0.f, 0.f};
        lds_head4<H>(t.a, v, av);
        if (kCombine) lds_head4<H>(t.b, v, bv);
        const float4 yv = reinterpret_cast<const float4*>(t.y)[v];
        const float4 nv = kNext ? reinterpret_cast<const float4*>(t.nz)[v] : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 xq = reinterpret_cast<const float4*>(t.x)[v];
        const uchar4 mv = reinterpret_cast<const uchar4*>(t.m)[v];
        float x[4] = {xq.x, xq.y, xq.z, xq.w}, o[4];
        const float y[4] = {yv.x, yv.y, yv.z, yv.w}, nz[4] = {nv.x, nv.y, nv.z, nv.w};
        const bool known[4] = {mv.x != 0, mv.y != 0, mv.z != 0, mv.w != 0};
#pragma unroll
        for (int j = 0; j < 4; ++j)
          boundary_element(av[j], bv[j], y[j], nz[j], known[j], x[j], o[j], kCombine, p.cfg, p.coef, true, kNext, rn, ry);
        const uint32_t i = e0 + 4 * v;
        if (p.out && i < p.out_end) st_f4(p.out + i, make_float4(o[0], o[1], o[2], o[3]), dead);
        *reinterpret_cast<float4*>(p.x + i) = make_float4(x[0], x[1], x[2], x[3]);
      }
    }
    __syncthreads();
    const uint32_t next = tile + (uint32_t)kStages * gridDim.x;
    if (threadIdx.x == 0 && next < tg.n_tiles) issue(next, s);
  }
}

template <typename H, bool kCombine, bool kNext>
int launch_boundary_tma(const BoundaryArgs& p, cudaStream_t s) {
  constexpr int kTile = 2048, kStages = 2;
  const int dev = current_device();
  const size_t smem = sizeof(BoundaryStage<H, kTile>) * kStages;
  static bool configured[kMaxDevices] = {};  // per instantiation of this launcher
  ensure_dynamic_smem(boundary_tma_kernel<H, kCombine, kNext, kTile, kStages>, smem, dev, configured);
  BTileGeom tg;
  tg.channels = p.g.per_row.d / p.g.spatial.d;
  tg.tiles_per_channel = (p.g.spatial.d + kTile - 1) / kTile;
  tg.n_tiles = (p.g.total / p.g.spatial.d) * tg.tiles_per_channel;
  unsigned grid = (unsigned)device_info(dev).sms * 2u;
  if (grid > tg.n_tiles) grid = tg.n_tiles;
  launch_kernel_smem(boundary_tma_kernel<H, kCombine, kNext, kTile, kStages>, dim3(grid), smem, s, p, tg);
  return check_launch();
}

// The LDG launch of the boundary kernel whose arguments are q (p: q's BoundaryArgs): packed or dense known bits,
// 4- or 1-wide vectors.  ldg_kernel names each kernel by its Args struct.
template <int N, typename H, bool kPk>
constexpr auto ldg_kernel(const BoundaryArgs&) { return boundary_kernel<N, H, kPk>; }

template <typename H, typename A>
int launch_ldg(const A& q, const BoundaryArgs& p, bool v4, cudaStream_t s) {
  const dim3 grid(blocks_for(v4 ? p.g.total / 4 : p.g.total));
  if (p.kwords) launch_kernel(v4 ? ldg_kernel<4, H, true>(q) : ldg_kernel<1, H, true>(q), grid, s, q);
  else launch_kernel(v4 ? ldg_kernel<4, H, false>(q) : ldg_kernel<1, H, false>(q), grid, s, q);
  return check_launch();
}

template <typename A>
int launch_ldg(const A& q, const BoundaryArgs& p, int dtype, bool v4, cudaStream_t s) {
  switch (dtype) {
    case LP_DTYPE_F32: return launch_ldg<float>(q, p, v4, s);
    case LP_DTYPE_BF16: return launch_ldg<__nv_bfloat16>(q, p, v4, s);
    default: return launch_ldg<__half>(q, p, v4, s);
  }
}

template <typename H>
int boundary_dispatch(const BoundaryArgs& p, bool v4, cudaStream_t s) {
  const bool tma = v4 && g_opt_tma != 0 && g_opt_tma_boundary != 0 && p.x && geometry_tma(p.g, p.mask) && p.g.total >= (uint32_t)g_opt_tma_min &&
                   aligned16(p.a) && (!p.combine || aligned16(p.b)) && aligned16(p.y) && aligned16(p.x) &&
                   (!p.next_table || aligned16(p.noise)) && (!p.out || aligned16(p.out));
  if (tma) {
    if (p.combine && p.next_table) return launch_boundary_tma<H, true, true>(p, s);
    if (p.combine) return launch_boundary_tma<H, true, false>(p, s);
    if (p.next_table) return launch_boundary_tma<H, false, true>(p, s);
    return launch_boundary_tma<H, false, false>(p, s);
  }
  return launch_ldg<H>(p, p, v4, s);
}

// what every boundary entry point rejects, before any CUDA call
static int boundary_check(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                          const lp_known* known, const float* x_inout, const float* out, const float* next_table) {
  if (!mo || !mo->a || !y || !mask) return LP_ERR_INVALID;
  if (known && (!known->words || !known->y || (next_table && !known->noise))) return LP_ERR_INVALID;
  if (!x_inout && !out) return LP_ERR_INVALID;
  if (next_table && (!noise || !x_inout)) return LP_ERR_INVALID;
  const int dtype = mo->dtype & ~LP_HEADS_DEAD;
  if (dtype != LP_DTYPE_F32 && dtype != LP_DTYPE_BF16 && dtype != LP_DTYPE_F16) return LP_ERR_INVALID;
  if (mo->combine && (dtype != LP_DTYPE_F32 || !mo->b || mo->b == mo->a)) return LP_ERR_INVALID;
  return LP_OK;
}

// Whether two of `bufs` -- fp32 buffers of `bytes` each but `out`, which spans out_bytes, NULL entries absent --
// share a byte.  A pair from the first `k` is exempt: the launch lets those alias, and with `whole` they may be one
// buffer but must not overlap in part (each element is read and written by one thread).
static bool aliased(std::initializer_list<const void*> bufs, size_t bytes, const void* out, size_t out_bytes, size_t k,
                    bool whole) {
  const void* const* v = bufs.begin();
  for (size_t m = 1; m < bufs.size(); ++m)
    for (size_t l = 0; l < m; ++l) {
      if (!v[m] || !v[l]) continue;
      const uintptr_t u = reinterpret_cast<uintptr_t>(v[m]), w = reinterpret_cast<uintptr_t>(v[l]);
      const size_t un = v[m] == out ? out_bytes : bytes, wn = v[l] == out ? out_bytes : bytes;
      const bool shared = u == w || (u < w + wn && w < u + un);
      if (m < k ? whole && shared && u != w : shared) return true;
    }
  return false;
}

// The setup every boundary entry point shares, before any CUDA call: the checks (the sampler's own are `valid`), the
// geometry, the aliasing rule on `states` (every fp32 buffer the launch reads or writes besides y and the noise, see
// aliased), the operands, whether the heads' lines may be dropped and whether the launch runs 4-wide.  `out` holds
// its first out_rows rows (out_rows < 0: every row).  An empty launch returns LP_OK with p.g.total == 0.
static int boundary_setup(BoundaryArgs& p, bool& v4, bool valid, const lp_heads* mo, const float* y, const float* noise,
                          const uint8_t* mask, const lp_known* known, float* x, float* out, int64_t out_rows,
                          float euler_coef, const float* next_table, const lp_dims* dims,
                          std::initializer_list<const void*> states, size_t k, bool whole = false) {
  v4 = false;
  if (int rc = boundary_check(mo, y, noise, mask, known, x, out, next_table)) return rc;
  if (!valid) return LP_ERR_INVALID;
  if (int rc = make_geometry(dims, p.g)) return rc;
  const uint32_t out_end = out_rows < 0 || (uint64_t)out_rows >= p.g.n_rows
                               ? p.g.total : (uint32_t)out_rows * p.g.per_row.d;
  const size_t bytes = (size_t)p.g.total * sizeof(float), out_bytes = (size_t)out_end * sizeof(float);
  if (aliased(states, bytes, out, out_bytes, k, whole)) return LP_ERR_INVALID;
  if (p.g.total == 0) return LP_OK;
  p.a = mo->a; p.b = mo->combine ? mo->b : nullptr; p.y = y; p.noise = noise; p.mask = mask; p.x = x;
  p.out = out_end ? out : nullptr;  // no row: the launch stores no out, as with out == NULL
  p.out_end = out_end;
  p.kwords = known ? known->words : nullptr; p.yk = known ? known->y : nullptr; p.nk = known ? known->noise : nullptr;
  p.next_table = next_table; p.cfg = mo->cfg; p.coef = euler_coef; p.combine = mo->combine != 0;
  p.l2 = l2_handoff(p.g.total);
  p.discard = heads_discard(mo, p.b, p.g.total, states, out, out_bytes);  // a dropped line holds no state
  const int dtype = mo->dtype & ~LP_HEADS_DEAD;
  v4 = geometry_vec4(p.g, p.mask) && head_aligned(p.a, dtype) && (!p.b || head_aligned(p.b, dtype)) &&
       aligned16(p.y) && (!p.noise || aligned16(p.noise));
  for (const void* b : states) v4 = v4 && (!b || aligned16(b));
  return LP_OK;
}

static int boundary_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                         const lp_known* known, float* x_inout, float* out, int64_t out_rows, float euler_coef,
                         const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  BoundaryArgs p;
  bool v4;
  if (int rc = boundary_setup(p, v4, true, mo, y, noise, mask, known, x_inout, out, out_rows, euler_coef, next_table,
                              dims, {x_inout, out}, 2))
    return rc;
  if (p.g.total == 0) return LP_OK;
  cudaStream_t s = (cudaStream_t)stream;
  switch (mo->dtype & ~LP_HEADS_DEAD) {
    case LP_DTYPE_F32: return boundary_dispatch<float>(p, v4, s);
    case LP_DTYPE_BF16: return boundary_dispatch<__nv_bfloat16>(p, v4, s);
    default: return boundary_dispatch<__half>(p, v4, s);
  }
}

// ---- the boundary of an outer step of a host-owned ancestral Euler loop ----------------------------------------
// k-diffusion's sample_euler_ancestral issues, after the wrapper call, sub, div, mul, add, randn_like, mul, mul, add
// as eight eager kernels; lp_boundary_ancestral does them in the boundary's one pass, each as the same correctly
// rounded fp32 operation, and draws the sampler's randn_like itself.
constexpr int kRngNone = -1;  // no rng: sigma_to == 0, the sampler takes no draw

struct AncestralArgs {
  BoundaryArgs b;  // x is never NULL; coef is unused
  lp_ancestral st;
  const float* tape0;
  const uint64_t* rng_state;
  uint64_t seed, draw0;
  uint32_t torch_T;  // threads of torch's randn grid (LP_RNG_TORCH)
};

// x += ((x - o) / sigma) down ; x += (xi s_noise) sigma_up
__device__ __forceinline__ void ancestral_update(float& x, float o, const lp_ancestral& st, bool draw, float xi) {
  x = __fadd_rn(x, __fmul_rn(__fdiv_rn(__fsub_rn(x, o), st.sigma), st.down));
  if (draw) x = __fadd_rn(x, __fmul_rn(__fmul_rn(xi, st.s_noise), st.sigma_up));
}

// per element: d = combine ? b + (a-b) cfg : a ; o = known ? y : d ; ancestral_update ; x = known ? rn n + ry y : x
__device__ __forceinline__ void ancestral_element(float a, float b, float y, float nz, bool known, float& x, float& o,
                                                  bool combine, float cfg, const lp_ancestral& st, bool draw, float xi,
                                                  bool next, float rn, float ry) {
  const float d = combine ? __fadd_rn(b, __fmul_rn(__fsub_rn(a, b), cfg)) : a;
  o = known ? y : d;
  ancestral_update(x, o, st, draw, xi);
  if (next) x = known ? fmaf(rn, nz, ry * y) : x;  // rounds as prologue_kernel does
}

// boundary_ancestral_kernel: x always read (where its update survives) and written.  No discard: with LP_RNG_TORCH a
// warp's elements are not one contiguous span, so a warp-span discard would drop lines other warps still read.
template <int N, bool kDraw>
struct AncestralUpdate {
  static constexpr bool kDiscard = false;
  const AncestralArgs& q;
  float xi[N];  // the sampler's randn_like at the vector's elements
  float xv[N] = {};
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t) {
    if (update) load_f<N>(q.b.x, i, xv);
  }
  __device__ __forceinline__ float& update(int j, float o) {
    ancestral_update(xv[j], o, q.st, kDraw, xi[j]);
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) { store_f<N>(q.b.x, i, xv); }
};

// LDG form: small or ragged launches, and the TAPE / PHILOX streams.  LP_RNG_TORCH maps threads onto torch's own
// randn grid: N == 4 as substep_torchvec_kernel does (thread (t, k) draws call k of subsequence t, a quad transposes
// its normals into four consecutive elements), N == 1 as advance_torch_kernel does.
template <int N, typename H, bool kPk, int kRng>
__global__ void __launch_bounds__(kBlock) boundary_ancestral_kernel(const AncestralArgs q) {
  pdl_prologue();
  const uint32_t total = q.b.g.total;
  if constexpr (kRng == LP_RNG_TORCH) {
    uint64_t seed = q.seed, o0 = q.draw0;
    if (q.rng_state) {
      seed = q.rng_state[0];
      o0 += q.rng_state[1];
    }
    const uint32_t T = q.torch_T;
    const uint32_t t = blockIdx.x * kBlock + threadIdx.x;  // torch thread == Philox subsequence
    if constexpr (N == 4) {
      const uint32_t k = blockIdx.y, l = t & 3u;
      const float4 n = torch_normal4(seed, o0, t, k);
      AncestralUpdate<4, true> u{q, {n.x, n.y, n.z, n.w}};
      quad_transpose(u.xi, l);
      const uint64_t e = (uint64_t)(t - l) + (uint64_t)(4u * k + l) * T;  // first of my 4 consecutive elements
      if (e >= total) return;
      boundary_vector<4, H, kPk>(q.b, (uint32_t)e, u);
    } else {
      if (t >= T) return;
      uint32_t call = 0;
      for (uint64_t base = t; base < total; base += 4ull * T, ++call) {
        const float4 n = torch_normal4(seed, o0, t, call);
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          const uint64_t li = base + (uint64_t)ii * T;
          if (li >= total) break;
          AncestralUpdate<1, true> u{q, {pick(n, ii)}};
          boundary_vector<1, H, kPk>(q.b, (uint32_t)li, u);
        }
      }
    }
  } else {
    const uint32_t i = (walk_index(q.b.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
    if (i >= total) return;
    AncestralUpdate<N, kRng != kRngNone> u{q, {}};
    float(&xi)[N] = u.xi;
    if constexpr (kRng == LP_RNG_TAPE) {
      load_f_ro<N>(q.tape0, i, xi);
    } else if constexpr (kRng == LP_RNG_PHILOX) {
      uint64_t seed = q.seed, d0 = q.draw0;
      if (q.rng_state) {
        seed = q.rng_state[0];
        d0 += q.rng_state[1];
      }
      const float4 n = philox_normal4(seed, d0, i >> 2);
      if constexpr (N == 4) {
        xi[0] = n.x; xi[1 % N] = n.y; xi[2 % N] = n.z; xi[3 % N] = n.w;
      } else {
        xi[0] = pick(n, i & 3);
      }
    }
    boundary_vector<N, H, kPk>(q.b, i, u);
  }
}

// LP_RNG_TORCH at HBM-bound sizes: the work-group form of substep_torch_tma_kernel (lp_substep.cu).  A group is
// (Philox call k, block b of kG consecutive subsequences) = four sub-tiles of kG consecutive elements, T apart; a
// producer warp streams each sub-tile's operand slices into its slot of a four-slot ring (full / empty mbarrier
// pairs) while the eight consumer warps draw; consumer thread c owns subsequences 4c..4c+3, so its four normals of a
// plane are one float4 of that plane's sub-tile.  One draw per launch.  kPk: the known bits and the packed y / noise
// spans (widened to 16-byte bounds) replace the dense y / noise slices and the uint8 mask slices.
template <typename H, int kG, bool kCombine, bool kNext, bool kPk>
struct __align__(128) AncestralSlot {
  H a[kG], b[kCombine ? kG : 8];  // every member starts on a 16-byte boundary (cp.async.bulk destinations)
  float x[kG];
  float y[kPk ? kG + 8 : kG];
  float nz[kNext ? (kPk ? kG + 8 : kG) : 4];
  uint8_t m[kPk ? 16 : kG];
  uint2 w[kPk ? kG / 32 : 2];
};

template <typename H, bool kCombine, bool kNext, bool kPk>
__global__ void __launch_bounds__(1024 / 4 + 32, 2)
    boundary_ancestral_torch_tma_kernel(const AncestralArgs q, const uint32_t groups_per_call, const uint32_t n_groups) {
  constexpr int kG = 1024, kConsumers = kG / 4;
  using Slot = AncestralSlot<H, kG, kCombine, kNext, kPk>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full[4], empty[4];
  Slot* slot = reinterpret_cast<Slot*>(smem_raw);
  pdl_prologue();
  const BoundaryArgs& p = q.b;
  const uint32_t T = q.torch_T, total = p.g.total;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      mbar_init(&full[j], 1);
      mbar_init(&empty[j], kConsumers);
    }
    mbar_fence_init();
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // first element / length of sub-tile j of group (k, b); a sub-tile past the end of the tensor is empty
  auto subtile = [&](uint32_t k, uint32_t b, int j, uint32_t& e0, uint32_t& len) {
    const uint64_t e = (uint64_t)(4u * k + (uint32_t)j) * T + (uint64_t)b * kG;
    if (e >= total) {
      e0 = 0;
      len = 0;
    } else {
      e0 = (uint32_t)e;
      len = total - e0 < (uint32_t)kG ? total - e0 : (uint32_t)kG;
    }
  };

  if (warp == kConsumers / 32) {  // ---------------- producer ----------------
    if (lane == 0) {
      const H* ap = static_cast<const H*>(p.a);
      const H* bp = static_cast<const H*>(p.b);
      const uint64_t dead = l2_policy_dead(p.l2);
      uint32_t it = 0;
      for (uint32_t step = blockIdx.x; step < n_groups; step += gridDim.x, ++it) {
        const uint32_t grp = walk_index(p.l2, step, n_groups);  // the consumers map `step` the same way
        const uint32_t k = grp / groups_per_call, b = grp - k * groups_per_call;
        uint32_t lo[4] = {0u, 0u, 0u, 0u}, hi[4] = {0u, 0u, 0u, 0u};
        if constexpr (kPk) {  // the packed spans of the group, read before the first slot wait, which hides them
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            uint32_t e0, len;
            subtile(k, b, j, e0, len);
            if (len) {
              lo[j] = __ldg(p.kwords + 2u * (e0 >> 5) + 1u);
              hi[j] = __ldg(p.kwords + 2u * ((e0 + len + 31u) >> 5) + 1u);
            }
          }
        }
#pragma unroll 1
        for (int j = 0; j < 4; ++j) {
          mbar_wait_relaxed(&empty[j], (it & 1u) ^ 1u);  // drained by the consumers (passes at once the first time)
          uint32_t e0, len;
          subtile(k, b, j, e0, len);
          const uint32_t fb = len * 4u, hb = len * (uint32_t)sizeof(H);
          const uint32_t heads = hb * (kCombine ? 2u : 1u);
          Slot& t = slot[j];
          if constexpr (kPk) {
            const uint32_t nw = (((len + 31u) >> 5) + 1u) & ~1u;  // whole words, an even number: 16-byte multiple
            const uint32_t ylo = (j == 0 ? lo[0] : j == 1 ? lo[1] : j == 2 ? lo[2] : lo[3]) & ~3u;
            const uint32_t yhi = ((j == 0 ? hi[0] : j == 1 ? hi[1] : j == 2 ? hi[2] : hi[3]) + 3u) & ~3u;
            const uint32_t yb = (yhi - ylo) * 4u;
            // an empty sub-tile still completes its phase: expect 0 bytes
            mbar_expect_tx(&full[j], len ? fb + heads + yb * (kNext ? 2u : 1u) + nw * 8u : 0u);
            if (len == 0) continue;
            tma_load_1d(t.a, ap + e0, hb, &full[j], dead);
            if (kCombine) tma_load_1d(t.b, bp + e0, hb, &full[j], dead);
            tma_load_1d(t.x, p.x + e0, fb, &full[j]);
            if (yb) tma_load_1d(t.y, p.yk + ylo, yb, &full[j]);
            if (kNext && yb) tma_load_1d(t.nz, p.nk + ylo, yb, &full[j]);
            tma_load_1d(t.w, p.kwords + 2u * (e0 >> 5), nw * 8u, &full[j]);
          } else {
            mbar_expect_tx(&full[j], fb * (kNext ? 3u : 2u) + heads + len);
            if (len == 0) continue;
            tma_load_1d(t.a, ap + e0, hb, &full[j], dead);
            if (kCombine) tma_load_1d(t.b, bp + e0, hb, &full[j], dead);
            tma_load_1d(t.x, p.x + e0, fb, &full[j]);
            tma_load_1d(t.y, p.y + e0, fb, &full[j]);
            if (kNext) tma_load_1d(t.nz, p.noise + e0, fb, &full[j]);
            // the mask is indexed per (row, channel): one slice per channel segment the sub-tile touches
            uint32_t e = e0, off = 0, rem = len;
            while (rem) {
              const uint32_t row = p.g.per_row.div(e);
              const uint32_t r = e - row * p.g.per_row.d;
              const uint32_t ch = p.g.spatial.div(r);
              const uint32_t s = r - ch * p.g.spatial.d;
              const uint32_t seg = rem < p.g.spatial.d - s ? rem : p.g.spatial.d - s;
              tma_load_1d(t.m + off, p.mask + row * p.g.mask_row_stride + ch * p.g.mask_channel_stride + s, seg,
                          &full[j]);
              e += seg;
              off += seg;
              rem -= seg;
            }
          }
        }
      }
    }
    return;
  }

  // ---------------- consumers ----------------
  uint64_t seed = q.seed, o0 = q.draw0;
  if (q.rng_state) {
    seed = q.rng_state[0];
    o0 += q.rng_state[1];
  }
  const uint32_t tid = threadIdx.x;  // vector index inside every sub-tile
  // one sub-tile's vector of this thread: slot -> registers, slot released, update, stores
  auto vector = [&](int j, uint32_t i, const float (&xi)[4]) {
    const Slot& t = slot[j];
    float a[4], b[4] = {0.f, 0.f, 0.f, 0.f}, y[4], nz[4] = {0.f, 0.f, 0.f, 0.f}, o[4];
    uint32_t kb;
    lds_head4<H>(t.a, tid, a);
    if (kCombine) lds_head4<H>(t.b, tid, b);
    const float4 xv = reinterpret_cast<const float4*>(t.x)[tid];
    if constexpr (kPk) {
      uint32_t idx;
      known_quad(t.w[tid >> 3], 4u * tid, kb, idx);
      idx -= t.w[0].y & ~3u;  // the spans start at the first word's base, rounded down
      gather_known4<true>(t.y, kb, idx, y);
      if (kNext) gather_known4<true>(t.nz, kb, idx, nz);
    } else {
      const float4 yv = reinterpret_cast<const float4*>(t.y)[tid];
      const uchar4 mv = reinterpret_cast<const uchar4*>(t.m)[tid];
      y[0] = yv.x; y[1] = yv.y; y[2] = yv.z; y[3] = yv.w;
      kb = (mv.x != 0 ? 1u : 0u) | (mv.y != 0 ? 2u : 0u) | (mv.z != 0 ? 4u : 0u) | (mv.w != 0 ? 8u : 0u);
      if (kNext) {
        const float4 nv = reinterpret_cast<const float4*>(t.nz)[tid];
        nz[0] = nv.x; nz[1] = nv.y; nz[2] = nv.z; nz[3] = nv.w;
      }
    }
    mbar_arrive(&empty[j]);  // this thread's reads of slot j are in registers: let it refill
    if (p.discard) {  // sub-tiles start on multiples of kG elements: a line below `total` lies in slot j
      discard_line<H>(p.a, i, total);
      if (kCombine) discard_line<H>(p.b, i, total);
    }
    float x[4] = {xv.x, xv.y, xv.z, xv.w};
    float rn = 0.f, ry = 0.f;
    if (kNext) {
      const uint32_t row = p.g.per_row.div(i);
      rn = __ldg(p.next_table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPN);
      ry = __ldg(p.next_table + (size_t)row * LP_TABLE_STRIDE + LP_T_REPY);
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
      ancestral_element(a[e], b[e], y[e], nz[e], ((kb >> e) & 1u) != 0, x[e], o[e], kCombine, p.cfg, q.st, true, xi[e],
                        kNext, rn, ry);
    if (p.out && i < p.out_end) st_f4(p.out + i, make_float4(o[0], o[1], o[2], o[3]), l2_policy_dead(p.l2));
    *reinterpret_cast<float4*>(p.x + i) = make_float4(x[0], x[1], x[2], x[3]);
  };
  uint32_t it = 0;
  for (uint32_t step = blockIdx.x; step < n_groups; step += gridDim.x, ++it) {
    const uint32_t grp = walk_index(p.l2, step, n_groups);
    const uint32_t k = grp / groups_per_call, b = grp - k * groups_per_call;
    const uint32_t t0 = b * kG + 4u * tid;  // my four Philox subsequences (torch threads)
    uint4 r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = torch_philox(seed, o0, t0 + i, k);
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // curand_normal4: planes 0,1 <- (x,y), planes 2,3 <- (z,w)
      float2 n[4];
#pragma unroll
      for (int i = 0; i < 4; i += 2)
        box_muller_curand_x2(h ? r[i].z : r[i].x, h ? r[i].w : r[i].y, h ? r[i + 1].z : r[i + 1].x,
                             h ? r[i + 1].w : r[i + 1].y, n[i], n[i + 1]);
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = 2 * h + jj;
        const float xi[4] = {jj ? n[0].y : n[0].x, jj ? n[1].y : n[1].x, jj ? n[2].y : n[2].x, jj ? n[3].y : n[3].x};
        mbar_wait(&full[j], it & 1u);
        uint32_t e0, len;
        subtile(k, b, j, e0, len);
        if (4u * tid < len) vector(j, e0 + 4u * tid, xi);
        else mbar_arrive(&empty[j]);
      }
    }
  }
}

template <typename H, bool kCombine, bool kNext, bool kPk>
int launch_ancestral_tma_cfg(const AncestralArgs& q, uint32_t calls, cudaStream_t s) {
  const int dev = current_device();
  const size_t smem = sizeof(AncestralSlot<H, 1024, kCombine, kNext, kPk>) * 4;
  const uint32_t groups_per_call = q.torch_T / 1024, n_groups = calls * groups_per_call;
  unsigned grid = (unsigned)device_info(dev).sms * 2u;
  if (grid > n_groups) grid = n_groups;
  static bool configured[kMaxDevices] = {};  // per instantiation of this launcher
  ensure_dynamic_smem(boundary_ancestral_torch_tma_kernel<H, kCombine, kNext, kPk>, smem, dev, configured);
  launch_kernel_ex(boundary_ancestral_torch_tma_kernel<H, kCombine, kNext, kPk>, dim3(grid), dim3(1024 / 4 + 32), smem,
                   s, q, groups_per_call, n_groups);
  return check_launch();
}

template <typename H, bool kCombine>
int launch_ancestral_tma(const AncestralArgs& q, bool packed, uint32_t calls, cudaStream_t s) {
  const bool next = q.b.next_table != nullptr;
  if (packed) {
    return next ? launch_ancestral_tma_cfg<H, kCombine, true, true>(q, calls, s)
                : launch_ancestral_tma_cfg<H, kCombine, false, true>(q, calls, s);
  }
  return next ? launch_ancestral_tma_cfg<H, kCombine, true, false>(q, calls, s)
              : launch_ancestral_tma_cfg<H, kCombine, false, false>(q, calls, s);
}

template <int N, typename H, int kRng>
void launch_ancestral_ldg(const AncestralArgs& q, dim3 grid, cudaStream_t s) {
  if (q.b.kwords) launch_kernel(boundary_ancestral_kernel<N, H, true, kRng>, grid, s, q);
  else launch_kernel(boundary_ancestral_kernel<N, H, false, kRng>, grid, s, q);
}

template <typename H>
int ancestral_dispatch(AncestralArgs& q, int mode, bool v4, cudaStream_t s) {
  const BoundaryArgs& p = q.b;
  const dim3 flat(v4 ? blocks_for(p.g.total / 4) : blocks_for(p.g.total));
  if (mode == LP_RNG_TORCH) {
    int64_t grid = 0;
    if (int rc = torch_grid(p.g.total, -1, &grid, nullptr)) return rc;
    q.torch_T = (uint32_t)(grid * 256);
    const uint64_t calls = ((uint64_t)p.g.total + 4ull * q.torch_T - 1) / (4ull * q.torch_T);
    // the torch-stream TMA sub-step's eligibility (lp_substep.cu)
    const bool tma = v4 && g_opt_tma != 0 && geometry_tma(p.g, p.mask) && p.g.total >= (uint32_t)g_opt_tma_min &&
                     aligned16(p.a) && (!p.combine || aligned16(p.b)) && aligned16(p.y) &&
                     (!p.next_table || aligned16(p.noise)) && q.torch_T % 1024 == 0 && p.g.spatial.d >= 64 &&
                     calls <= 0xffffffffull / 4;
    if (tma) {
      const bool packed = p.kwords && aligned16(p.kwords) && aligned16(p.yk) && (!p.next_table || aligned16(p.nk));
      if constexpr (sizeof(H) == 4) {  // the CFG combine needs fp32 heads
        if (p.combine) return launch_ancestral_tma<H, true>(q, packed, (uint32_t)calls, s);
      }
      return launch_ancestral_tma<H, false>(q, packed, (uint32_t)calls, s);
    }
    if (v4 && calls <= 65535) launch_ancestral_ldg<4, H, LP_RNG_TORCH>(q, dim3((unsigned)grid, (unsigned)calls), s);
    else launch_ancestral_ldg<1, H, LP_RNG_TORCH>(q, dim3((unsigned)grid), s);
  } else if (mode == LP_RNG_TAPE) {
    if (v4 && aligned16(q.tape0)) launch_ancestral_ldg<4, H, LP_RNG_TAPE>(q, flat, s);
    else launch_ancestral_ldg<1, H, LP_RNG_TAPE>(q, dim3(blocks_for(p.g.total)), s);
  } else if (mode == LP_RNG_PHILOX) {
    if (v4) launch_ancestral_ldg<4, H, LP_RNG_PHILOX>(q, flat, s);
    else launch_ancestral_ldg<1, H, LP_RNG_PHILOX>(q, flat, s);
  } else {
    if (v4) launch_ancestral_ldg<4, H, kRngNone>(q, flat, s);
    else launch_ancestral_ldg<1, H, kRngNone>(q, flat, s);
  }
  return check_launch();
}

static int boundary_ancestral_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                                   const lp_known* known, float* x_inout, float* out, int64_t out_rows,
                                   const lp_ancestral* step,
                                   const lp_rng* rng, const float* next_table, const lp_dims* dims,
                                   lp_stream_t stream) {
  const int mode = rng ? rng->mode : kRngNone;
  const bool valid = x_inout && step && step->sigma > 0.f && (rng || step->sigma_up == 0.f) &&
                     (!rng || mode == LP_RNG_TAPE || mode == LP_RNG_PHILOX || mode == LP_RNG_TORCH) &&
                     (mode != LP_RNG_TAPE || rng->tape0);
  AncestralArgs q;
  bool v4;
  if (int rc = boundary_setup(q.b, v4, valid, mo, y, noise, mask, known, x_inout, out, out_rows, 0.f, next_table, dims,
                              {x_inout, out}, 2))
    return rc;
  if (q.b.g.total == 0) return LP_OK;
  q.st = *step;
  q.tape0 = rng ? rng->tape0 : nullptr;
  q.rng_state = rng ? rng->state : nullptr;
  q.seed = rng ? rng->seed : 0;
  q.draw0 = rng ? rng->draw0 : 0;
  q.torch_T = 0;
  cudaStream_t s = (cudaStream_t)stream;
  switch (mo->dtype & ~LP_HEADS_DEAD) {
    case LP_DTYPE_F32: return ancestral_dispatch<float>(q, mode, v4, s);
    case LP_DTYPE_BF16: return ancestral_dispatch<__nv_bfloat16>(q, mode, v4, s);
    default: return ancestral_dispatch<__half>(q, mode, v4, s);
  }
}

// ---- the boundary of an outer step of a host-owned DPM-Solver++(2M) loop --------------------------------------
// k-diffusion's sample_dpmpp_2m issues, after the wrapper call, mul, mul, sub (first order) or mul, mul, sub, mul, mul,
// sub (second order) as eager kernels, with per-step 0-d tensors the host hands in as lp_multistep;
// lp_boundary_multistep does them in the boundary's one pass, each as the same correctly rounded fp32 operation.
struct MultistepArgs {
  BoundaryArgs b;  // x is never NULL; coef is unused
  lp_multistep st;
  const float* old;  // the previous step's out; NULL: first-order step
};

// dd = old ? c_cur o - c_old old : o ; x = ratio x - em1 dd ; x and old read where x's update survives
template <int N>
struct MultistepUpdate {
  static constexpr bool kDiscard = true;
  const MultistepArgs& q;
  float xv[N] = {}, dv[N] = {};
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t dead) {
    if (update) load_f<N>(q.b.x, i, xv);
    if (q.old && update) load_head_ro<N, float>(q.old, i, dv, dead);  // nothing reads the previous out again
  }
  __device__ __forceinline__ float& update(int j, float o) {
    const float dd = q.old ? __fsub_rn(__fmul_rn(q.st.c_cur, o), __fmul_rn(q.st.c_old, dv[j])) : o;
    xv[j] = __fsub_rn(__fmul_rn(q.st.ratio, xv[j]), __fmul_rn(q.st.em1, dd));
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) { store_f<N>(q.b.x, i, xv); }
};

template <int N, typename H, bool kPk>
__global__ void __launch_bounds__(kBlock) boundary_multistep_kernel(const MultistepArgs q) {
  pdl_prologue();
  const uint32_t i = (walk_index(q.b.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
  if (i >= q.b.g.total) return;
  MultistepUpdate<N> u{q};
  boundary_vector<N, H, kPk>(q.b, i, u);
}

template <int N, typename H, bool kPk>
constexpr auto ldg_kernel(const MultistepArgs&) { return boundary_multistep_kernel<N, H, kPk>; }

static int boundary_multistep_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                                   const lp_known* known, float* x_inout, float* out, const float* old_out,
                                   const lp_multistep* step, const float* next_table, const lp_dims* dims,
                                   lp_stream_t stream) {
  MultistepArgs q;
  bool v4;
  // the launch writes x and out while it reads old_out
  if (int rc = boundary_setup(q.b, v4, x_inout && step, mo, y, noise, mask, known, x_inout, out, -1, 0.f, next_table, dims,
                              {x_inout, out, old_out}, 2))
    return rc;
  if (q.b.g.total == 0) return LP_OK;
  q.st = *step;
  q.old = old_out;
  return launch_ldg(q, q.b, mo->dtype & ~LP_HEADS_DEAD, v4, (cudaStream_t)stream);
}

// ---- the boundary of a wrapper call of a host-owned DPM-Solver-2 loop ------------------------------------------
// k-diffusion's sample_dpm_2 issues, after each wrapper call, sub, div, mul, add as eager kernels, with per-step 0-d
// tensors the host hands in as lp_midpoint; lp_boundary_midpoint does them in the boundary's one pass, each as the
// same correctly rounded fp32 operation.
struct MidpointArgs {
  BoundaryArgs b;       // b.x is x_out; coef is unused
  lp_midpoint st;
  const float* xin;
  const float* xbase;   // == xin: read once
  int evict;            // x_in / x_base are not read again before a whole network call: load them evict-first
};

// x_out = base + ((in - o) / sigma) dt ; x_in and x_base read where x_out's update survives, x_out not read
template <int N>
struct MidpointUpdate {
  static constexpr bool kDiscard = true;
  const MidpointArgs& q;
  float iv[N] = {}, sv[N] = {}, xv[N];
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t dead) {
    if (!update) return;
    const uint64_t xp = q.evict ? dead : 0;
    load_f<N>(q.xin, i, iv, xp);
    if (q.xbase != q.xin) {
      load_f<N>(q.xbase, i, sv, xp);
    } else {
#pragma unroll
      for (int j = 0; j < N; ++j) sv[j] = iv[j];
    }
  }
  __device__ __forceinline__ float& update(int j, float o) {
    xv[j] = __fadd_rn(sv[j], __fmul_rn(__fdiv_rn(__fsub_rn(iv[j], o), q.st.sigma), q.st.dt));
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) {
    store_f<N>(q.b.x, i, xv);  // normal policy: the next network call reads x_out first
  }
};

template <int N, typename H, bool kPk>
__global__ void __launch_bounds__(kBlock) boundary_midpoint_kernel(const MidpointArgs q) {
  pdl_prologue();
  const uint32_t i = (walk_index(q.b.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
  if (i >= q.b.g.total) return;
  MidpointUpdate<N> u{q};
  boundary_vector<N, H, kPk>(q.b, i, u);
}

template <int N, typename H, bool kPk>
constexpr auto ldg_kernel(const MidpointArgs&) { return boundary_midpoint_kernel<N, H, kPk>; }

static int boundary_midpoint_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                                  const lp_known* known, const float* x_in, const float* x_base, float* x_out,
                                  float* out, int64_t out_rows, const lp_midpoint* step, const float* next_table, const lp_dims* dims,
                                  lp_stream_t stream) {
  MidpointArgs q;
  bool v4;
  // one thread reads and writes each element: the three states are each one buffer or disjoint, and out, which the
  // launch writes, shares no byte with any of them
  if (int rc = boundary_setup(q.b, v4, step && x_in && x_base && x_out, mo, y, noise, mask, known, x_out, out,
                              out_rows, 0.f, next_table, dims, {x_in, x_base, x_out, out}, 3, true))
    return rc;
  if (q.b.g.total == 0) return LP_OK;
  q.st = *step;
  q.xin = x_in;
  q.xbase = x_base;
  q.evict = !(x_in == x_out && x_base == x_out);  // the predictor's X, the corrector's X2 and X
  return launch_ldg(q, q.b, mo->dtype & ~LP_HEADS_DEAD, v4, (cudaStream_t)stream);
}

// ---- the boundary of an outer step of a host-owned DEIS loop ---------------------------------------------------
// ComfyUI's sample_deis issues, after the wrapper call, sub, div, then mul, add per term of its multistep sum (left to
// right) as eager kernels, with fp32 coefficients the host hands in as lp_deis; lp_boundary_deis does them in the
// boundary's one pass, each as the same correctly rounded fp32 operation, and keeps d for the next two steps.
struct DeisArgs {
  BoundaryArgs b;      // x is never NULL; coef is unused
  lp_deis st;
  float* dout;         // NULL: no later step reads this step's d
  const float* p1;     // the previous step's d; NULL: first order
  const float* p2;     // the one before it; NULL: first or second order
};

// d = (x - o) / sigma ; x = x + c_cur d [+ c_prev1 p1 [+ c_prev2 p2]] ; the history read where x's update survives,
// x also where d is written at a known position
template <int N>
struct DeisUpdate {
  static constexpr bool kDiscard = true;
  const DeisArgs& q;
  const bool second = q.p1 != nullptr, third = q.p2 != nullptr;
  float xv[N] = {}, v1[N] = {}, v2[N] = {}, dv[N];
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t dead) {
    if (update || q.dout) load_f<N>(q.b.x, i, xv);
    if (second && update) load_f_ro<N>(q.p1, i, v1);                  // the next step reads it again, as its d_prev2
    if (third && update) load_head_ro<N, float>(q.p2, i, v2, dead);   // nothing reads it again
  }
  __device__ __forceinline__ float& update(int j, float o) {
    dv[j] = __fdiv_rn(__fsub_rn(xv[j], o), q.st.sigma);
    float u = __fadd_rn(xv[j], __fmul_rn(q.st.c_cur, dv[j]));
    if (second) u = __fadd_rn(u, __fmul_rn(q.st.c_prev1, v1[j]));
    if (third) u = __fadd_rn(u, __fmul_rn(q.st.c_prev2, v2[j]));
    xv[j] = u;
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) {
    if (q.dout) store_f<N>(q.dout, i, dv);  // normal policy: the next step reads it
    store_f<N>(q.b.x, i, xv);
  }
};

template <int N, typename H, bool kPk>
__global__ void __launch_bounds__(kBlock) boundary_deis_kernel(const DeisArgs q) {
  pdl_prologue();
  const uint32_t i = (walk_index(q.b.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
  if (i >= q.b.g.total) return;
  DeisUpdate<N> u{q};
  boundary_vector<N, H, kPk>(q.b, i, u);
}

template <int N, typename H, bool kPk>
constexpr auto ldg_kernel(const DeisArgs&) { return boundary_deis_kernel<N, H, kPk>; }

static int boundary_deis_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                              const lp_known* known, float* x_inout, float* out, int64_t out_rows, float* d_out, const float* d_prev1,
                              const float* d_prev2, const lp_deis* step, const float* next_table, const lp_dims* dims,
                              lp_stream_t stream) {
  DeisArgs q;
  bool v4;
  // the launch writes x, out and d_out while it reads the history: the three histories share no byte with each other
  // or with x and out
  if (int rc = boundary_setup(q.b, v4, x_inout && step && (d_prev1 || !d_prev2), mo, y, noise, mask, known, x_inout,
                              out, out_rows, 0.f, next_table, dims, {x_inout, out, d_out, d_prev1, d_prev2}, 2))
    return rc;
  if (q.b.g.total == 0) return LP_OK;
  q.st = *step;
  q.dout = d_out;
  q.p1 = d_prev1;
  q.p2 = d_prev2;
  return launch_ldg(q, q.b, mo->dtype & ~LP_HEADS_DEAD, v4, (cudaStream_t)stream);
}

// ---- the boundary of an outer step of a host-owned gradient-estimation loop ---------------------------------------
// ComfyUI's sample_gradient_estimation issues, after the wrapper call, sub, div, then mul, add (the Euler step) and,
// from its second step on, sub, mul, mul, add (the correction), with scalars the host hands in as
// lp_gradient_estimation; lp_boundary_gradient_estimation does them in the boundary's one pass, each as the same
// correctly rounded fp32 operation, and keeps d for the next step.
struct GeArgs {
  BoundaryArgs b;      // x is never NULL; coef is unused
  lp_gradient_estimation st;
  float* dout;         // NULL: no later step reads this step's d
  const float* prev;   // the previous step's d; NULL: no correction
};

// d = (x - o) / sigma ; x = final ? o : x + d dt [+ (gm1 (d - prev)) dt] ; the history read where x's update
// survives, x where the update reads it or d is written
template <int N>
struct GeUpdate {
  static constexpr bool kDiscard = true;
  const GeArgs& q;
  float xv[N] = {}, pv[N] = {}, dv[N];
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t dead) {
    if ((update && !q.st.final) || q.dout) load_f<N>(q.b.x, i, xv);
    if (q.prev && update) load_head_ro<N, float>(q.prev, i, pv, dead);  // nothing reads it again
  }
  __device__ __forceinline__ float& update(int j, float o) {
    dv[j] = __fdiv_rn(__fsub_rn(xv[j], o), q.st.sigma);
    float u = o;
    if (!q.st.final) {
      u = __fadd_rn(xv[j], __fmul_rn(dv[j], q.st.dt));
      if (q.prev) u = __fadd_rn(u, __fmul_rn(__fmul_rn(q.st.gm1, __fsub_rn(dv[j], pv[j])), q.st.dt));
    }
    xv[j] = u;
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) {
    if (q.dout) store_f<N>(q.dout, i, dv);  // normal policy: the next step reads it
    store_f<N>(q.b.x, i, xv);
  }
};

template <int N, typename H, bool kPk>
__global__ void __launch_bounds__(kBlock) boundary_ge_kernel(const GeArgs q) {
  pdl_prologue();
  const uint32_t i = (walk_index(q.b.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
  if (i >= q.b.g.total) return;
  GeUpdate<N> u{q};
  boundary_vector<N, H, kPk>(q.b, i, u);
}

template <int N, typename H, bool kPk>
constexpr auto ldg_kernel(const GeArgs&) { return boundary_ge_kernel<N, H, kPk>; }

static int boundary_ge_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                            const lp_known* known, float* x_inout, float* out, int64_t out_rows, float* d_out, const float* d_prev,
                            const lp_gradient_estimation* step, const float* next_table, const lp_dims* dims,
                            lp_stream_t stream) {
  GeArgs q;
  bool v4;
  // the launch writes x, out and d_out while it reads d_prev: the four share no byte
  if (int rc = boundary_setup(q.b, v4, x_inout && step && !(step->final && d_prev), mo, y, noise, mask, known, x_inout,
                              out, out_rows, 0.f, next_table, dims, {x_inout, out, d_out, d_prev}, 0))
    return rc;
  if (q.b.g.total == 0) return LP_OK;
  q.st = *step;
  q.dout = d_out;
  q.prev = d_prev;
  return launch_ldg(q, q.b, mo->dtype & ~LP_HEADS_DEAD, v4, (cudaStream_t)stream);
}

// ---- the boundary of the second wrapper call of a host-owned Heun loop ------------------------------------------
// k-diffusion's sample_heun issues, after its second wrapper call, sub, div (d_2), add, div by 2, mul, add as eager
// kernels, with d from its first call and per-step 0-d tensors the host hands in as lp_heun; lp_boundary_heun does
// them in the boundary's one pass, each as the same correctly rounded fp32 operation, and recomputes d from x and the
// first call's denoised latent with the sampler's sub, div.
struct HeunArgs {
  BoundaryArgs b;       // b.x is x, read and written; coef is unused
  lp_heun st;
  const float* x2;      // the state the second call ran on
  const float* prev;    // the first call's out
};

// d = (x - prev) / sigma ; d2 = (x2 - o) / sigma_next ; x = x + ((d + d2) * 0.5) dt ; x, x2 and the first call's out
// read where x's update survives
template <int N>
struct HeunUpdate {
  static constexpr bool kDiscard = true;
  const HeunArgs& q;
  float xv[N] = {}, v2[N] = {}, pv[N] = {};
  __device__ __forceinline__ void load(uint32_t i, bool update, uint64_t dead) {
    if (!update) return;
    load_f<N>(q.b.x, i, xv);
    load_head_ro<N, float>(q.x2, i, v2, dead);    // the next predictor overwrites it unread
    load_head_ro<N, float>(q.prev, i, pv, dead);  // so does the next first call
  }
  __device__ __forceinline__ float& update(int j, float o) {
    const float d = __fdiv_rn(__fsub_rn(xv[j], pv[j]), q.st.sigma);
    const float d2 = __fdiv_rn(__fsub_rn(v2[j], o), q.st.sigma_next);
    // torch divides by the Python scalar 2 as a multiply by 0.5: the same bits, there being no flush to zero
    xv[j] = __fadd_rn(xv[j], __fmul_rn(__fmul_rn(__fadd_rn(d, d2), 0.5f), q.st.dt));
    return xv[j];
  }
  __device__ __forceinline__ void store(uint32_t i) {
    store_f<N>(q.b.x, i, xv);  // normal policy: the next network call reads x first
  }
};

template <int N, typename H, bool kPk>
__global__ void __launch_bounds__(kBlock) boundary_heun_kernel(const HeunArgs q) {
  pdl_prologue();
  const uint32_t i = (walk_index(q.b.l2, blockIdx.x, gridDim.x) * kBlock + threadIdx.x) * N;
  if (i >= q.b.g.total) return;
  HeunUpdate<N> u{q};
  boundary_vector<N, H, kPk>(q.b, i, u);
}

template <int N, typename H, bool kPk>
constexpr auto ldg_kernel(const HeunArgs&) { return boundary_heun_kernel<N, H, kPk>; }

static int boundary_heun_impl(const lp_heads* mo, const float* y, const float* noise, const uint8_t* mask,
                              const lp_known* known, float* x, const float* x2, const float* out_prev, float* out,
                              const lp_heun* step, const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  HeunArgs q;
  bool v4;
  // the launch writes x and out while it reads x2 and out_prev: the four share no byte
  if (int rc = boundary_setup(q.b, v4, step && x && x2 && out_prev, mo, y, noise, mask, known, x, out, -1, 0.f, next_table,
                              dims, {x, x2, out_prev, out}, 0))
    return rc;
  if (q.b.g.total == 0) return LP_OK;
  q.st = *step;
  q.x2 = x2;
  q.prev = out_prev;
  return launch_ldg(q, q.b, mo->dtype & ~LP_HEADS_DEAD, v4, (cudaStream_t)stream);
}

// ---- un-fused OU advance (advance_time_overdamped, lanpaint.py:232-254) --------
struct AdvanceArgs {
  float* x;
  const float* c;
  const uint8_t* mask;
  const float* table;
  const float* tape0;
  const uint64_t* rng_state;
  uint64_t seed, draw0;
  Geometry g;
  uint32_t torch_T;
  int half;
};

__device__ __forceinline__ float advance_element(float x, float c, bool known, float xi,
                                                 const float* __restrict__ t, int half) {
  const float* k = t + (known ? LP_T_CLS1 : LP_T_CLS0);
  const float e = __ldg(k + (half ? LP_C_EH : LP_C_EF));
  const float kk = __ldg(k + (half ? LP_C_KH : LP_C_KF));
  const float sd = __ldg(k + (half ? LP_C_SH : LP_C_SF));
  const float xt = x * __ldg(t + LP_T_INVS);
  return fmaf(e, xt, fmaf(kk, c, sd * xi)) * __ldg(t + LP_T_S);
}

template <int kRng>
__global__ void __launch_bounds__(kBlock) advance_kernel(const AdvanceArgs a) {
  pdl_prologue();
  const uint32_t i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= a.g.total) return;
  uint32_t row, mi;
  locate(a.g, i, row, mi);
  float xi;
  if (kRng == LP_RNG_TAPE) {
    xi = __ldg(a.tape0 + i);
  } else {
    uint64_t seed = a.seed, d0 = a.draw0;
    if (a.rng_state) {
      seed = a.rng_state[0];
      d0 += a.rng_state[1];
    }
    xi = pick(philox_normal4(seed, d0, i >> 2), i & 3);
  }
  a.x[i] = advance_element(a.x[i], __ldg(a.c + i), __ldg(a.mask + mi) != 0, xi,
                           a.table + (size_t)row * LP_TABLE_STRIDE, a.half);
}

__global__ void __launch_bounds__(kBlock) advance_torch_kernel(const AdvanceArgs a) {
  pdl_prologue();
  const uint32_t T = a.torch_T;
  const uint32_t tid = blockIdx.x * kBlock + threadIdx.x;
  if (tid >= T) return;
  uint64_t seed = a.seed, o0 = a.draw0;
  if (a.rng_state) {
    seed = a.rng_state[0];
    o0 += a.rng_state[1];
  }
  uint32_t call = 0;
  for (uint64_t base = tid; base < a.g.total; base += 4ull * T, ++call) {
    const float4 n1 = torch_normal4(seed, o0, tid, call);
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const uint64_t li = base + (uint64_t)ii * T;
      if (li >= a.g.total) break;
      const uint32_t i = (uint32_t)li;
      uint32_t row, mi;
      locate(a.g, i, row, mi);
      a.x[i] = advance_element(a.x[i], __ldg(a.c + i), __ldg(a.mask + mi) != 0, pick(n1, ii),
                               a.table + (size_t)row * LP_TABLE_STRIDE, a.half);
    }
  }
}

// ---- early-stop statistics: two masked sums of squared differences ---------------
// Grid-stride over float4 groups; per-thread partials -> warp shuffle -> one smem slot per warp ->
// one atomicAdd(double) per block per sum (earlystop.py:51-55 _weighted_mse numerators).
struct StatsArgs {
  const float* a;
  const float* b;
  const uint8_t* mask;
  const uint8_t* ring;
  const float* table;
  double* sums;
  Geometry g;
};

template <int N>
__global__ void __launch_bounds__(kBlock) stop_stats_kernel(const StatsArgs s) {
  pdl_prologue();
  float acc_in = 0.f, acc_ring = 0.f;
  const uint32_t stride = gridDim.x * kBlock * N;
  for (uint32_t i = (blockIdx.x * kBlock + threadIdx.x) * N; i < s.g.total; i += stride) {
    uint32_t row, mi;
    locate(s.g, i, row, mi);
    float av[N], bv[N];
    bool known[N], on_ring[N];
    load_f_ro<N>(s.a, i, av);
    load_f_ro<N>(s.b, i, bv);
    load_m<N>(s.mask, mi, known);
    if (s.ring) {
      load_m<N>(s.ring, mi, on_ring);
    } else {
#pragma unroll
      for (int j = 0; j < N; ++j) on_ring[j] = false;
    }
    const float scale = s.table ? __ldg(s.table + (size_t)row * LP_TABLE_STRIDE + LP_T_INVS) : 1.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      const float d = (av[j] - bv[j]) * scale;
      const float d2 = d * d;
      acc_in += known[j] ? 0.f : d2;
      acc_ring += on_ring[j] ? d2 : 0.f;
    }
  }
  __shared__ float part[2][kBlock / 32];
  acc_in = warp_sum(acc_in);
  acc_ring = warp_sum(acc_ring);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) {
    part[0][w] = acc_in;
    part[1][w] = acc_ring;
  }
  __syncthreads();
  if (w == 0) {
    float u = lane < kBlock / 32 ? part[0][lane] : 0.f;
    float v = lane < kBlock / 32 ? part[1][lane] : 0.f;
    u = warp_sum(u);
    v = warp_sum(v);
    if (lane == 0) {
      atomicAdd(s.sums + 0, (double)u);
      atomicAdd(s.sums + 1, (double)v);
    }
  }
}

}  // namespace lp

using namespace lp;

extern "C" int lp_prologue_f32(const float* x, const float* y, const float* noise, const uint8_t* mask,
                               float* x_model, float* x_copy, const float* table, const lp_dims* dims,
                               lp_stream_t stream) {
  if (!x || !y || !noise || !mask || !x_model || !table) return LP_ERR_INVALID;
  Geometry g;
  if (int rc = make_geometry(dims, g)) return rc;
  if (g.total == 0) return LP_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const bool v4 = geometry_vec4(g, mask) && aligned16(x) && aligned16(y) && aligned16(noise) &&
                  aligned16(x_model) && (!x_copy || aligned16(x_copy));
  if (v4) launch_kernel(prologue_kernel<4>, dim3(blocks_for(g.total / 4)), s, x, y, noise, mask, x_model, x_copy, table, g);
  else launch_kernel(prologue_kernel<1>, dim3(blocks_for(g.total)), s, x, y, noise, mask, x_model, x_copy, table, g);
  return check_launch();
}

extern "C" int lp_boundary(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                           float* x_inout, float* out, float euler_coef, const float* next_table, const lp_dims* dims,
                           lp_stream_t stream) {
  return boundary_impl(model_out, y, noise, mask, nullptr, x_inout, out, -1, euler_coef, next_table, dims, stream);
}

extern "C" int lp_boundary_known(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                 const lp_known* known, float* x_inout, float* out, float euler_coef,
                                 const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  if (!known) return LP_ERR_INVALID;
  return boundary_impl(model_out, y, noise, mask, known, x_inout, out, -1, euler_coef, next_table, dims, stream);
}

extern "C" int lp_boundary_known_rows(const lp_heads* model_out, const float* y, const float* noise,
                                      const uint8_t* mask, const lp_known* known, float* x_inout, float* out,
                                      int64_t out_rows, float euler_coef, const float* next_table, const lp_dims* dims,
                                      lp_stream_t stream) {
  if (!known || out_rows < 0) return LP_ERR_INVALID;
  return boundary_impl(model_out, y, noise, mask, known, x_inout, out, out_rows, euler_coef, next_table, dims, stream);
}

extern "C" int lp_boundary_ancestral(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                     const lp_known* known, float* x_inout, float* out, const lp_ancestral* step,
                                     const lp_rng* rng, const float* next_table, const lp_dims* dims,
                                     lp_stream_t stream) {
  return boundary_ancestral_impl(model_out, y, noise, mask, known, x_inout, out, -1, step, rng, next_table, dims,
                                 stream);
}

extern "C" int lp_boundary_ancestral_rows(const lp_heads* model_out, const float* y, const float* noise,
                                          const uint8_t* mask, const lp_known* known, float* x_inout, float* out,
                                          int64_t out_rows, const lp_ancestral* step, const lp_rng* rng,
                                          const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  if (out_rows < 0) return LP_ERR_INVALID;
  return boundary_ancestral_impl(model_out, y, noise, mask, known, x_inout, out, out_rows, step, rng, next_table, dims,
                                 stream);
}

extern "C" int lp_boundary_multistep(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                     const lp_known* known, float* x_inout, float* out, const float* old_out,
                                     const lp_multistep* step, const float* next_table, const lp_dims* dims,
                                     lp_stream_t stream) {
  return boundary_multistep_impl(model_out, y, noise, mask, known, x_inout, out, old_out, step, next_table, dims,
                                 stream);
}

extern "C" int lp_boundary_midpoint(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                    const lp_known* known, const float* x_in, const float* x_base, float* x_out,
                                    float* out, const lp_midpoint* step, const float* next_table, const lp_dims* dims,
                                    lp_stream_t stream) {
  return boundary_midpoint_impl(model_out, y, noise, mask, known, x_in, x_base, x_out, out, -1, step, next_table, dims,
                                stream);
}

extern "C" int lp_boundary_midpoint_rows(const lp_heads* model_out, const float* y, const float* noise,
                                         const uint8_t* mask, const lp_known* known, const float* x_in,
                                         const float* x_base, float* x_out, float* out, int64_t out_rows,
                                         const lp_midpoint* step, const float* next_table, const lp_dims* dims,
                                         lp_stream_t stream) {
  if (out_rows < 0) return LP_ERR_INVALID;
  return boundary_midpoint_impl(model_out, y, noise, mask, known, x_in, x_base, x_out, out, out_rows, step, next_table,
                                dims, stream);
}

extern "C" int lp_boundary_deis(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                const lp_known* known, float* x_inout, float* out, float* d_out, const float* d_prev1,
                                const float* d_prev2, const lp_deis* step, const float* next_table, const lp_dims* dims,
                                lp_stream_t stream) {
  return boundary_deis_impl(model_out, y, noise, mask, known, x_inout, out, -1, d_out, d_prev1, d_prev2, step,
                            next_table, dims, stream);
}

extern "C" int lp_boundary_deis_rows(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                     const lp_known* known, float* x_inout, float* out, int64_t out_rows, float* d_out,
                                     const float* d_prev1, const float* d_prev2, const lp_deis* step,
                                     const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  if (out_rows < 0) return LP_ERR_INVALID;
  return boundary_deis_impl(model_out, y, noise, mask, known, x_inout, out, out_rows, d_out, d_prev1, d_prev2, step,
                            next_table, dims, stream);
}

extern "C" int lp_boundary_gradient_estimation(const lp_heads* model_out, const float* y, const float* noise,
                                               const uint8_t* mask, const lp_known* known, float* x_inout, float* out,
                                               float* d_out, const float* d_prev, const lp_gradient_estimation* step,
                                               const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  return boundary_ge_impl(model_out, y, noise, mask, known, x_inout, out, -1, d_out, d_prev, step, next_table, dims,
                          stream);
}

extern "C" int lp_boundary_gradient_estimation_rows(const lp_heads* model_out, const float* y, const float* noise,
                                                    const uint8_t* mask, const lp_known* known, float* x_inout,
                                                    float* out, int64_t out_rows, float* d_out, const float* d_prev,
                                                    const lp_gradient_estimation* step, const float* next_table,
                                                    const lp_dims* dims, lp_stream_t stream) {
  if (out_rows < 0) return LP_ERR_INVALID;
  return boundary_ge_impl(model_out, y, noise, mask, known, x_inout, out, out_rows, d_out, d_prev, step, next_table,
                          dims, stream);
}

extern "C" int lp_boundary_heun(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                const lp_known* known, float* x, const float* x2, const float* out_prev, float* out,
                                const lp_heun* step, const float* next_table, const lp_dims* dims, lp_stream_t stream) {
  return boundary_heun_impl(model_out, y, noise, mask, known, x, x2, out_prev, out, step, next_table, dims, stream);
}

extern "C" int lp_epilogue_f32(const float* model_out, const float* y, const uint8_t* mask, float* out,
                               const lp_dims* dims, lp_stream_t stream) {
  if (!out) return LP_ERR_INVALID;
  lp_heads h = {model_out, nullptr, LP_DTYPE_F32, 0, 0.f, 0.f};
  return boundary_impl(&h, y, nullptr, mask, nullptr, nullptr, out, -1, 0.f, nullptr, dims, stream);
}

extern "C" int lp_epilogue_euler_f32(const float* model_out, const float* y, const uint8_t* mask, float* x_inout,
                                     float* out, float euler_coef, const lp_dims* dims, lp_stream_t stream) {
  if (!x_inout) return LP_ERR_INVALID;
  lp_heads h = {model_out, nullptr, LP_DTYPE_F32, 0, 0.f, 0.f};
  return boundary_impl(&h, y, nullptr, mask, nullptr, x_inout, out, -1, euler_coef, nullptr, dims, stream);
}

extern "C" int lp_step_boundary_f32(const float* model_out, const float* y, const float* noise, const uint8_t* mask,
                                    float* x_inout, float* out, float euler_coef, const float* next_table,
                                    const lp_dims* dims, lp_stream_t stream) {
  if (!noise || !x_inout || !next_table) return LP_ERR_INVALID;
  lp_heads h = {model_out, nullptr, LP_DTYPE_F32, 0, 0.f, 0.f};
  return boundary_impl(&h, y, noise, mask, nullptr, x_inout, out, -1, euler_coef, next_table, dims, stream);
}

extern "C" int lp_epilogue_cfg_f32(const float* cond, const float* uncond, float cfg, const float* y,
                                   const uint8_t* mask, float* x_inout, float* out, float euler_coef,
                                   const lp_dims* dims, lp_stream_t stream) {
  if (!cond || !uncond || !out) return LP_ERR_INVALID;
  lp_heads h = {cond, uncond, LP_DTYPE_F32, 1, cfg, cfg};
  return boundary_impl(&h, y, nullptr, mask, nullptr, x_inout, out, -1, euler_coef, nullptr, dims, stream);
}

extern "C" int lp_advance_f32(float* x_model, const float* c_state, const uint8_t* mask, const float* table,
                              const lp_dims* dims, const lp_rng* rng, int half, lp_stream_t stream) {
  if (!x_model || !c_state || !mask || !table || !rng) return LP_ERR_INVALID;
  AdvanceArgs a;
  if (int rc = make_geometry(dims, a.g)) return rc;
  if (a.g.total == 0) return LP_OK;
  a.x = x_model; a.c = c_state; a.mask = mask; a.table = table; a.tape0 = rng->tape0;
  a.rng_state = rng->state; a.seed = rng->seed; a.draw0 = rng->draw0; a.torch_T = 0; a.half = half != 0;
  cudaStream_t s = (cudaStream_t)stream;
  if (rng->mode == LP_RNG_TORCH) {
    int64_t grid = 0;
    if (int rc = torch_grid(a.g.total, -1, &grid, nullptr)) return rc;
    a.torch_T = (uint32_t)(grid * 256);
    launch_kernel(advance_torch_kernel, dim3((unsigned)grid), s, a);
  } else if (rng->mode == LP_RNG_TAPE) {
    if (!rng->tape0) return LP_ERR_INVALID;
    launch_kernel(advance_kernel<LP_RNG_TAPE>, dim3(blocks_for(a.g.total)), s, a);
  } else if (rng->mode == LP_RNG_PHILOX) {
    launch_kernel(advance_kernel<LP_RNG_PHILOX>, dim3(blocks_for(a.g.total)), s, a);
  } else {
    return LP_ERR_INVALID;
  }
  return check_launch();
}

extern "C" int lp_stop_stats_f32(const float* a, const float* b, const uint8_t* mask, const uint8_t* ring,
                                 const float* table, const lp_dims* dims, double* sums, lp_stream_t stream) {
  if (!a || !b || !mask || !sums) return LP_ERR_INVALID;
  StatsArgs s;
  if (int rc = make_geometry(dims, s.g)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaMemsetAsync(sums, 0, 2 * sizeof(double), st) != cudaSuccess) {
    check_launch();
    return LP_ERR_CUDA;
  }
  if (s.g.total == 0) return LP_OK;
  s.a = a; s.b = b; s.mask = mask; s.ring = ring; s.table = table; s.sums = sums;
  const int sms = device_info(current_device()).sms;
  const bool v4 = geometry_vec4(s.g, mask) && aligned16(a) && aligned16(b) && (!ring || aligned4(ring));
  const uint32_t groups = v4 ? s.g.total / 4 : s.g.total;
  unsigned grid = blocks_for(groups);
  const unsigned cap = (unsigned)sms * 8;  // persistent-sized: 8 CTAs of 256 threads per SM
  if (grid > cap) grid = cap;
  if (v4) launch_kernel(stop_stats_kernel<4>, dim3(grid), st, s);
  else launch_kernel(stop_stats_kernel<1>, dim3(grid), st, s);
  return check_launch();
}

/*
 * lanpaint_b200 -- C ABI of the H100-native (sm_90a) LanPaint Langevin hot path.
 *
 * The reference (scraed/LanPaint) is pure Python/PyTorch and has no FFI; this
 * header is the boundary a maintainer would bind (ctypes stub in
 * INTEGRATION.md).  Each entry point names the reference code it replaces,
 * paths relative to the reference root.
 *
 * Conventions
 *   - all tensors are fp32, contiguous, NC(T)HW; "per_sample" = C*spatial
 *   - the mask is uint8, 1 = known / keep (the reference's latent_mask,
 *     src/LanPaint/nodes.py:281-283), either full shape or [B,1,spatial]
 *     broadcast over channels (mask_channel_stride = 0)
 *   - per-sample scalars live in a device "coefficient table" of
 *     LP_TABLE_STRIDE floats per row, built on the host by
 *     lp_build_coef_table() -- this removes every exp/expm1/sqrt/where and
 *     every host sync of src/LanPaint/lanpaint.py:205,232-254,295-328 from
 *     the per-element path
 *   - every device entry point is asynchronous on the caller's stream, does
 *     not allocate, does not synchronise, is CUDA-graph capturable and
 *     re-entrant; it returns an lp_status (never throws)
 */
#ifndef LANPAINT_B200_H_
#define LANPAINT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LP_ABI_VERSION 5
/* Backward-compatible additions within LP_ABI_VERSION: 1 = LP_HEADS_DEAD (a dtype bit every earlier library
 * rejected with LP_ERR_INVALID, so no earlier caller can have set it); 2 = lp_multistep and
 * lp_boundary_multistep (a new entry point: nothing an earlier caller binds changes).  Later entry points
 * (lp_midpoint and lp_boundary_midpoint, lp_deis and lp_boundary_deis, lp_gradient_estimation and
 * lp_boundary_gradient_estimation, lp_heun and lp_boundary_heun, the row-bounded lp_boundary_*_rows forms) leave
 * LP_ABI_MINOR at 2: a caller detects one by its symbol, which is how lanpaint_b200._native binds every entry point
 * (by name). */
#define LP_ABI_MINOR 2
#define LP_TABLE_STRIDE 32 /* floats per table row (one 128-byte line), layout below */

typedef void* lp_stream_t; /* a cudaStream_t / CUstream */

typedef enum lp_status {
  LP_OK = 0,
  LP_ERR_INVALID = 1,   /* null pointer / negative size / bad flag combination */
  LP_ERR_ALIGNMENT = 2, /* reserved: all paths fall back to scalar access instead */
  LP_ERR_CUDA = 3,      /* launch failed; see lp_last_cuda_error() */
  LP_ERR_UNSUPPORTED = 4
} lp_status;

/* Table row layout (floats).  Class 0 = free / regenerate region ("x branch",
 * mask 0), class 1 = known region ("y branch", mask 1).
 *   0 c_tgt      sqrt(abt)/(1-abt)          coefficient of the score target in C
 *   1 S          model-space x = x_t * S    (VE: sqrt(1+sigma^2); flow: 1/(sqrt(abt)+sqrt(1-abt)))
 *   2 inv_S
 *   3 lam        Lambda
 *   4 one_plus_lam
 *   5 rep_noise  replace step: known = rep_noise*noise + rep_y*y
 *   6 rep_y
 *   7 corr       audio target correction c (1 = none)         [lanpaint.py:173-180]
 *   8+8k .. 15+8k  class k: g (= A - 1/(1-abt)), dt, e_full, k_full, sd_full, e_half, k_half, sd_half
 *   24,25      sdm[k]   = sqrt((e_half sd_half)^2 + sd_half^2): std of the two half-advance kicks a steady
 *                         fused launch applies, merged into one Gaussian (LP_SUBSTEP_MERGE_NOISE)
 *   26,27      sdmf[k]  = sqrt((e_half sd_full)^2 + sd_half^2): same for the FIRST|FUSE_NEXT launch
 *   28..31     reserved (0)
 * where for an advance over h:  e = exp(-A h), k = (1-e)/A, sd = sqrt(D^2 (1-exp(-2 A h))/(2A)), D = sqrt(2)
 * (src/LanPaint/lanpaint.py:232-254), full = dt, half = dt/2.
 */
enum {
  LP_T_CTGT = 0, LP_T_S = 1, LP_T_INVS = 2, LP_T_LAM = 3, LP_T_ONEPLAM = 4,
  LP_T_REPN = 5, LP_T_REPY = 6, LP_T_CORR = 7, LP_T_CLS0 = 8, LP_T_CLS1 = 16, LP_T_SDM = 24, LP_T_SDMF = 26,
  LP_C_G = 0, LP_C_DT = 1, LP_C_EF = 2, LP_C_KF = 3, LP_C_SF = 4, LP_C_EH = 5, LP_C_KH = 6, LP_C_SH = 7
};

/* Engine hyper-parameters: constructor of the reference engine,
 * src/LanPaint/lanpaint.py:8-21. */
typedef struct lp_hyper {
  double step_size;     /* StepSize */
  double lam;           /* Lambda */
  double beta;          /* Beta */
  double min_step_frac; /* MinStepFrac */
  int32_t flow;         /* IS_FLUX or IS_FLOW */
  int32_t reserved;
} lp_hyper;

typedef struct lp_dims {
  int64_t n_rows;              /* table rows == samples B (or B*2 with the audio class split) */
  int64_t per_row;             /* elements per table row (C*spatial for one sample) */
  int64_t spatial;             /* elements per channel */
  int64_t mask_row_stride;     /* mask elements between consecutive rows */
  int64_t mask_channel_stride; /* 0 = mask broadcast over channels, spatial = full-shape mask */
  int64_t row_split;           /* 0 = off.  > 0: positions >= row_split inside every row use table row
                                  (n_rows + row) instead of (row): the MiniMax-H3 flat pack, whose trailing
                                  audio positions run on their own sigma schedule (lanpaint.py:60-74); the
                                  table then holds 2*n_rows rows */
} lp_dims;

/* How the Gaussian draws of src/LanPaint/lanpaint.py:252 (torch.randn_like on
 * the global generator) are supplied. */
typedef enum lp_rng_mode {
  LP_RNG_TAPE = 0,   /* caller passes the draws as tensors (exact CPU-oracle parity) */
  LP_RNG_PHILOX = 1, /* in-kernel Philox4x32-10, element i <- component i&3 of counter (i>>2, draw) */
  LP_RNG_TORCH = 2   /* in-kernel Philox reproducing torch.randn_like's CUDA stream bit for bit */
} lp_rng_mode;

typedef struct lp_rng {
  int32_t mode;          /* lp_rng_mode */
  int32_t reserved;
  const float* tape0;    /* TAPE: draw consumed first by the launch */
  const float* tape1;    /* TAPE: draw consumed second (may be NULL if unused) */
  uint64_t seed;         /* PHILOX/TORCH */
  uint64_t draw0;        /* PHILOX: draw index; TORCH: philox offset of the first draw */
  uint64_t draw1;        /* second draw index / offset */
  const uint64_t* state; /* optional device pointer {seed, base}: if non-NULL, seed is read from
                            it and base is added to draw0/draw1 (lets a captured CUDA graph be
                            replayed with a fresh stream position) */
} lp_rng;

/* Element type of the model's output tensors ("heads").  State, clean latent, noise and all arithmetic are
 * fp32 like the reference's (its autocast(float32) wrappers, lanpaint.py:201,239); a network that returns
 * bf16 / fp16 predictions is read as is and widened in registers -- the same values the reference gets from
 * type promotion when it subtracts an fp32 x_t from them (lanpaint.py:182-184) -- instead of paying a
 * separate .float() pass (6 B/element read + 8 B/element written per head pair). */
typedef enum lp_dtype { LP_DTYPE_F32 = 0, LP_DTYPE_BF16 = 1, LP_DTYPE_F16 = 2 } lp_dtype;

/* lp_heads.dtype may carry this bit next to the lp_dtype: nothing reads a or b after the launch.  The HBM-bound
 * update kernels (the TMA-staged sub-steps, the LDG step boundary, the TMA-staged ancestral boundary) then drop
 * every 128-byte line of the heads they have finished reading from the L2 without writing it back
 * (discard.global.L2): a network's output is still dirty in L2 when the update that consumes it starts, and its
 * write-back is HBM traffic nothing needs.  Afterwards the heads' memory holds undefined values until it is written
 * again.  A launch ignores the bit unless both heads start on a 128-byte boundary and no output of the launch
 * overlaps them; option "discard_heads" 0 ignores it everywhere.  Results do not depend on it. */
enum { LP_HEADS_DEAD = 0x100 };

/* The model's prediction(s) for one call, as the kernels consume them (src/LanPaint/lanpaint.py:34-43,
 * 159-171; src/LanPaint/nodes.py:161-175):
 *   combine == 0   a = x0, b = x0_BIG (NULL or == a: the two heads alias)
 *   combine != 0   a = cond, b = uncond (raw network outputs); the kernel forms
 *                  x0 = b + (a - b)*cfg and x0_BIG = b + (a - b)*cfg_big in registers with the eager
 *                  sub/mul/add roundings (requires dtype == LP_DTYPE_F32 so that they ARE the eager roundings) */
typedef struct lp_heads {
  const void* a;
  const void* b;
  int32_t dtype;   /* lp_dtype of a and b, optionally | LP_HEADS_DEAD */
  int32_t combine;
  float cfg, cfg_big;
} lp_heads;

/* ---- library ---------------------------------------------------------- */
int lp_abi_version(void);
const char* lp_status_string(int status);
int lp_last_cuda_error(void); /* cudaError_t of the last failed launch on this thread */
/* Process-wide switches (also read once from the environment: LANPAINT_B200_PDL, LANPAINT_B200_TMA,
 * LANPAINT_B200_TMA_MIN, LANPAINT_B200_TMA_BOUNDARY, LANPAINT_B200_L2_HANDOFF):
 *   "pdl" 1|0      programmatic dependent launch on every kernel (default 1)
 *   "tma" 1|0      use the TMA-staged persistent variants (cp.async.bulk + mbarrier ring) of the fused sub-step
 *                  (philox and torch streams) and of the step-boundary kernel when eligible: spatial a multiple
 *                  of 16, no side outputs, no row split (default 1; 2..5 select alternative tile geometries of
 *                  the philox kernel, for measurement)
 *   "tma_min"      smallest launch, in elements, that takes a TMA-staged variant (default 2^18)
 *   "tma_boundary" 1|0  lp_boundary: TMA-staged kernel when eligible | always the LDG kernel (default 0: measured
 *                  faster inside a job, where the network's output is still in L2)
 *   "l2_handoff"   bits, for measurement: 1 the TMA sub-steps and the step-boundary kernels walk their launch
 *                  tail-first, 2 evict-first L2 policy on the heads, C and the boundary's output (default 3);
 *                  launches of fewer than 2^20 elements, whose job stays in L2, use neither.  Results do not
 *                  depend on it.
 *   "discard_heads" 1|0  honour LP_HEADS_DEAD (default 1; 0 for measurement) */
int lp_set_option(const char* name, int value);

/* Host-only self test of the index arithmetic the kernels rely on (the multiply-shift division that
 * replaces `/` and `%` by per_row and spatial): returns the number of (n, d) pairs, out of `samples`
 * pseudo-random ones plus every edge case, for which it disagrees with n / d.  0 = sound. */
int64_t lp_selftest_index_math(int64_t samples);

/* Device self test of the two-lane Box-Muller the torch-stream kernels use: runs it next to the scalar cuRAND
 * form on `n` pseudo-random input quadruples (plus 4096 edge cases: extremes of u and v, u == 1) and counts bitwise
 * mismatches into *mismatches_dev (a device uint64, zeroed by the call).  0 = the two are interchangeable. */
int lp_selftest_box_muller(int64_t n, uint64_t seed, unsigned long long* mismatches_dev, lp_stream_t stream);

/* Device self test of the LP_RNG_PHILOX Box-Muller (MUFU lg2 / sqrt / sin / cos) over all 2^32 values of one input
 * word: the first word (sweep_second == 0) or the second, the other held at fixed_word.  *nonfinite_dev (a device
 * uint64) receives the number of inputs with a non-finite output and *max_err_dev (a device double) the largest
 * |fast - fp64 Box-Muller| over both outputs, the fp64 transform taken of the same fp32 u and v.  Both are zeroed by
 * the call. */
int lp_selftest_normal_fast(uint32_t fixed_word, int sweep_second, unsigned long long* nonfinite_dev,
                            double* max_err_dev, lp_stream_t stream);

/* ---- host: coefficient table ------------------------------------------- */
/* Replaces LanPaint.prepare_step_size + the mask blend of A/D/dt + the
 * exp/expm1/where/sqrt of advance_time_overdamped (lanpaint.py:81,205-214,
 * 232-254,295-328).  Inputs are the reference's own per-sample fp32 values
 * (abt, VE sigma: nodes.py:242-252) widened to double; arithmetic is fp64,
 * results rounded once to fp32.  rep_noise/rep_y may be NULL (-> 0, 1);
 * corr may be NULL (-> 1).  table_out: n_rows*LP_TABLE_STRIDE floats (host). */
int lp_build_coef_table(const double* abt, const double* ve_sigma, const double* rep_noise,
                        const double* rep_y, const double* corr, int64_t n_rows,
                        const lp_hyper* hyper, float* table_out);

/* Same table from explicit per-row half time steps (the `dtx/2`, `dty/2` a caller of the reference's
 * `langevin_dynamics(x_t, score, mask, step_size, current_times, sigma_x, sigma_y)` controls directly,
 * lanpaint.py:192,301-302).  scale = S per row (NULL: 1, i.e. the state stays in VP space).
 * target_is_x0e != 0: the kernels' x0 and y inputs both carry x_t + score (an arbitrary score callback's
 * result), so the known-region target must pass through unchanged (lam = 0 inside the target only). */
int lp_build_coef_table_dt(const double* abt, const double* scale, const double* dt_free,
                           const double* dt_known, double lam, int32_t target_is_x0e, int64_t n_rows,
                           float* table_out);

/* Geometry of torch's CUDA randn kernel (ATen/native/cuda/DistributionTemplates.h:
 * calc_execution_policy) for `numel` elements on `device`: grid blocks of 256
 * threads and the philox offset increment one draw consumes. */
int lp_torch_randn_geometry(int64_t numel, int device, int64_t* grid_out, uint64_t* increment_out);

/* ---- device: hot path --------------------------------------------------- */
/* mask_f32 > 0.5 -> uint8 (the binarise of nodes.py:281-283, done once). */
int lp_pack_mask_f32(const float* mask_f32, uint8_t* mask_u8, int64_t n, int invert, lp_stream_t stream);

/* The known-operand layout.  The clean latent y and the noise image are only ever read at known positions
 * (lanpaint.py:85-94,151-154,182-184), and both are constant for a whole job, so the kernels that stream them
 * can read them packed: only their known elements, in element order.  Over the flat element index i of the
 * latent (total = n_rows * per_row elements), with W = ceil(total / 32):
 *   words[2w]     known bits of elements 32w .. 32w+31 (bit b <-> element 32w + b; 0 past the end)
 *   words[2w + 1] number of known elements before element 32w, i.e. the packed index of the first known one
 *   words[2W], words[2W + 1] = 0, number of known elements (end sentinel)
 * so a known element i sits at packed index words[2w+1] + popc(words[2w] & ((1 << (i & 31)) - 1)), w = i >> 5.
 * The bits follow the uint8 mask through its strides, so a channel-broadcast mask and a full-shape one give the
 * same layout.  words holds lp_known_words(total) uint32 (the tail is the builder's scratch); y_known and
 * noise_known hold total + 4 floats (the TMA-staged kernels fetch 16-byte aligned spans that may reach 3 floats
 * past the last known element). */
typedef struct lp_known {
  const uint32_t* words;
  const float* y;     /* y at known elements */
  const float* noise; /* the noise image at known elements (NULL: not packed; a boundary that needs it fails) */
} lp_known;

int64_t lp_known_words(int64_t total);

/* Builds words, y_known and (if noise != NULL) noise_known from the uint8 mask and the dense operands: three
 * small launches, once per job.  Reads the mask through dims like every other entry point. */
int lp_pack_known(const uint8_t* mask, const lp_dims* dims, const float* y, const float* noise, uint32_t* words,
                  float* y_known, float* noise_known, lp_stream_t stream);

/* Replace step + change of variables, lanpaint.py:85-99:
 *   x_model = mask ? rep_noise*noise + rep_y*y : x
 * written to x_model (may alias x) and, if non-NULL, x_copy. */
int lp_prologue_f32(const float* x, const float* y, const float* noise, const uint8_t* mask,
                    float* x_model, float* x_copy, const float* table, const lp_dims* dims,
                    lp_stream_t stream);

/* Flags of lp_substep_f32. */
enum {
  LP_SUBSTEP_FIRST = 1,     /* sub-step 0: no previous C, one full-dt advance (run_overdamped, args is None) */
  LP_SUBSTEP_FUSE_NEXT = 2, /* also apply the first half-advance of the NEXT sub-step (uses the new C) */
  LP_SUBSTEP_STORE_C = 4,   /* write the new C even without FUSE_NEXT (un-fused / early-stop loops) */
  LP_SUBSTEP_MERGE_NOISE = 8 /* with FUSE_NEXT and LP_RNG_PHILOX only: the two Gaussian kicks of the launch are
                                independent and nothing observes the state between them, so draw ONE normal with
                                the summed variance (table sdm/sdmf).  Same Markov chain in distribution, half the
                                RNG work; not stream-compatible with the reference, hence never used by TAPE/TORCH */
};

/* One fused Langevin launch = everything between two model calls
 * (lanpaint.py:113-142 -> langevin_dynamics :192-293 -> score_model :159-184,
 * Coef_C :217-220, advance_time_overdamped :232-254, run_overdamped :274-286):
 *   post-model half of sub-step i  [FIRST: C=Coef_C(x); x=adv(x,dt,C)
 *                                   else : Cn=Coef_C(x); x+=(Cn-C)dt; x=adv(x,dt/2,C_old)]
 *   + pre-model half of sub-step i+1 [x=adv(x,dt/2,Cn)] when FUSE_NEXT.
 * x_model is read (the model's input) and overwritten with the next model
 * input; c_state is read (unless FIRST) and written (FUSE_NEXT or STORE_C);
 * x0/x0_big are the model's two heads (x0_big NULL or == x0: aliased);
 * x_copy (optional) also receives the new x (the reference's
 * input_x.copy_(x), lanpaint.py:156); x0e_out (optional) receives
 * x_t + score, the LangevinState.x0 the early stopper watches.
 * Consumes 2 draws with FUSE_NEXT (1 with MERGE_NOISE), else 1. */
int lp_substep_f32(float* x_model, const float* x0, const float* x0_big, const float* y,
                   const uint8_t* mask, float* c_state, float* x_copy, float* x0e_out,
                   const float* table, const lp_dims* dims, const lp_rng* rng, int flags,
                   lp_stream_t stream);

/* The general form of lp_substep_f32: heads of any lp_dtype, optionally the two classifier-free-guidance
 * combines folded in (lp_heads).  lp_substep_f32 / lp_substep_cfg_f32 are this call with fp32 heads. */
int lp_substep(float* x_model, const lp_heads* heads, const float* y, const uint8_t* mask, float* c_state,
               float* x_copy, float* x0e_out, const float* table, const lp_dims* dims, const lp_rng* rng,
               int flags, lp_stream_t stream);

/* lp_substep with the known-operand layout of the same y and mask (lp_pack_known).  The TMA-staged torch-stream
 * kernel then fetches the packed y and the known bits instead of the dense y and the uint8 mask; every other
 * kernel reads the dense operands, which must stay valid.  Results are bit-identical to lp_substep. */
int lp_substep_known(float* x_model, const lp_heads* heads, const float* y, const uint8_t* mask, const lp_known* known,
                     float* c_state, float* x_copy, float* x0e_out, const float* table, const lp_dims* dims,
                     const lp_rng* rng, int flags, lp_stream_t stream);

/* lp_substep_f32 with the two classifier-free-guidance combines folded in (SURVEY 8f rank 1; replaces the
 * two cfg_function calls of sampling_function_LanPaint, src/LanPaint/nodes.py:175): the caller passes the
 * network's raw cond / uncond x0 predictions and the two scales,
 *   x0 = uncond + (cond - uncond) * cfg ;   x0_big = uncond + (cond - uncond) * cfg_big
 * evaluated with the same three roundings as the eager sub/mul/add, so results equal the unfused path bit
 * for bit.  Same bytes read as lp_substep_f32; saves the 2 x 3 element-wise kernels and 2 tensors of
 * traffic the combines cost per model call. */
int lp_substep_cfg_f32(float* x_model, const float* cond, const float* uncond, float cfg, float cfg_big,
                       const float* y, const uint8_t* mask, float* c_state, float* x_copy, float* x0e_out,
                       const float* table, const lp_dims* dims, const lp_rng* rng, int flags,
                       lp_stream_t stream);

/* The un-fused building block: one exact OU advance of the model-space state,
 *   x_t = x/S;  x_t = e x_t + k C + sd xi;  x = x_t S
 * over dt (half = 0) or dt/2 (half = 1) -- advance_time_overdamped,
 * lanpaint.py:232-254.  Consumes 1 draw (rng->draw0 / tape0). */
int lp_advance_f32(float* x_model, const float* c_state, const uint8_t* mask, const float* table,
                   const lp_dims* dims, const lp_rng* rng, int half, lp_stream_t stream);

/* out = mask ? y : model_out   (lanpaint.py:151-154). */
int lp_epilogue_f32(const float* model_out, const float* y, const uint8_t* mask, float* out,
                    const lp_dims* dims, lp_stream_t stream);

/* lp_epilogue_f32 fused with the update k-diffusion's Euler sampler applies right after it
 * (sample_euler: d = (x - denoised)/sigma; x = x + d*(sigma_next - sigma)), for hosts that own the
 * sampler loop (SURVEY 8f rank 3):
 *   out = mask ? y : model_out ;  x = x + (x - out) * euler_coef      euler_coef = (sigma_next - sigma)/sigma
 * x_inout is the model-space state lp_substep_f32 left behind (the rewritten sampler x).  out may be NULL when
 * nobody reads the denoised latent (no preview callback): the pass then writes only x. */
int lp_epilogue_euler_f32(const float* model_out, const float* y, const uint8_t* mask, float* x_inout,
                          float* out, float euler_coef, const lp_dims* dims, lp_stream_t stream);

/* The boundary between two outer steps of a host-owned Euler loop in ONE pass: epilogue of step s
 * (lanpaint.py:151-154), k-diffusion's Euler update, and the replace step of step s+1 (lanpaint.py:85-94,
 * coefficients rep_noise/rep_y of `next_table`):
 *   out = mask ? y : model_out ;  x = x + (x - out)*euler_coef ;  x = mask ? rep_n*noise + rep_y*y : x
 * Known positions never read x or model_out; free positions never read noise.  out may be NULL. */
int lp_step_boundary_f32(const float* model_out, const float* y, const float* noise, const uint8_t* mask,
                         float* x_inout, float* out, float euler_coef, const float* next_table,
                         const lp_dims* dims, lp_stream_t stream);

/* The general boundary of an outer step, everything after its last model call in ONE pass
 * (lanpaint.py:151-157, k-diffusion sample_euler, lanpaint.py:85-94 of the next step):
 *   d   = model_out->combine ? b + (a - b)*cfg : a                      (heads of any lp_dtype)
 *   out = mask ? y : d                                                  written when out != NULL
 *   x   = x + (x - out)*euler_coef                                      when x_inout != NULL
 *   x   = mask ? rep_noise*noise + rep_y*y : x  (row of next_table)     when next_table != NULL (needs noise, x_inout)
 * lp_epilogue_f32, lp_epilogue_euler_f32, lp_step_boundary_f32 and lp_epilogue_cfg_f32 are special cases. */
int lp_boundary(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask, float* x_inout,
                float* out, float euler_coef, const float* next_table, const lp_dims* dims, lp_stream_t stream);

/* lp_boundary with the known-operand layout (lp_pack_known; known->noise is needed when next_table != NULL): the
 * LDG kernel reads the known bits and the packed y / noise instead of the uint8 mask and the dense y / noise.
 * The TMA-staged kernel (option "tma_boundary") keeps the dense operands.  Bit-identical to lp_boundary. */
int lp_boundary_known(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                      const lp_known* known, float* x_inout, float* out, float euler_coef, const float* next_table,
                      const lp_dims* dims, lp_stream_t stream);

/* Row-bounded `out`.  Each lp_boundary_*_rows entry point is the entry point of the same name without the suffix,
 * except that `out` is stored only for the first out_rows rows (elements < out_rows * per_row): out then needs room
 * for min(out_rows, n_rows) rows only, and no byte past them is written.  out_rows >= n_rows is the entry point itself,
 * out_rows == 0 stores no out, like out == NULL, and out_rows < 0 is LP_ERR_INVALID.  Every other store, x included,
 * and which heads' lines are dropped (LP_HEADS_DEAD) are unchanged.  A host whose denoised latent is read only by a
 * preview of the first request passes 1.  (lp_boundary_multistep and lp_boundary_heun have no such form: the host
 * reads their out back whole in a later launch.) */
int lp_boundary_known_rows(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                           const lp_known* known, float* x_inout, float* out, int64_t out_rows, float euler_coef,
                           const float* next_table, const lp_dims* dims, lp_stream_t stream);

/* One outer step of k-diffusion's sample_euler_ancestral, as the host precomputes it (get_ancestral_step in Python
 * doubles, then one rounding to fp32 per field). */
typedef struct lp_ancestral {
  float sigma;    /* sigma_from: d = (x - out) / sigma */
  float down;     /* (float)(sigma_down - sigma_from), the difference taken in double */
  float s_noise;  /* multiplies the draw first ... */
  float sigma_up; /* ... then this (0 when eta == 0: the draw is still taken) */
} lp_ancestral;

/* The boundary of an outer step of a host-owned ANCESTRAL Euler loop in ONE pass: lp_boundary_known with the Euler
 * update replaced by sample_euler_ancestral's, the sampler's own torch.randn_like(x) drawn inside the kernel:
 *   d   = model_out->combine ? b + (a - b)*cfg : a
 *   out = mask ? y : d                                                  written when out != NULL
 *   x   = x + ((x - out) / sigma) * down
 *   x   = x + (xi * s_noise) * sigma_up                                 when rng != NULL; xi = the launch's draw
 *   x   = mask ? rep_noise*noise + rep_y*y : x  (row of next_table)     when next_table != NULL
 * Every operation of the update is the single correctly rounded fp32 operation the eager sampler issues (sub, div,
 * mul, add; never contracted), so x equals the un-fused route's bit for bit.  The sampler draws exactly when
 * sigma_to > 0, also when eta == 0 makes sigma_up zero: the caller passes rng exactly then (draw0 / tape0 only).
 * rng == NULL: no draw, no stream position consumed.  known may be NULL (dense y / noise / mask).  With
 * LP_RNG_TORCH an HBM-bound launch takes a TMA-staged kernel of the torch-stream sub-step's work-group form; every
 * other launch takes an LDG kernel.  Results do not depend on which. */
int lp_boundary_ancestral(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                          const lp_known* known, float* x_inout, float* out, const lp_ancestral* step,
                          const lp_rng* rng, const float* next_table, const lp_dims* dims, lp_stream_t stream);
/* lp_boundary_ancestral with a row-bounded out (see lp_boundary_known_rows). */
int lp_boundary_ancestral_rows(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                               const lp_known* known, float* x_inout, float* out, int64_t out_rows,
                               const lp_ancestral* step, const lp_rng* rng, const float* next_table,
                               const lp_dims* dims, lp_stream_t stream);

/* One outer step of k-diffusion's sample_dpmpp_2m (DPM-Solver++(2M)), with t = -log(sigma) and h = t_next - t.  The
 * host evaluates these with the sampler's own torch expressions on the schedule, on the device the sampler runs on,
 * and reads them back: they are the fp32 scalars the sampler multiplies with. */
typedef struct lp_multistep {
  float ratio; /* sigma_fn(t_next) / sigma_fn(t), sigma_fn(t) = exp(-t): 0 on the step to sigma = 0 */
  float em1;   /* expm1(-h): -1 on the step to sigma = 0 */
  float c_cur; /* 1 + 1/(2r), r = h_last / h: weight of this step's denoised latent (second-order steps) */
  float c_old; /* 1/(2r): weight of the previous step's denoised latent (second-order steps) */
} lp_multistep;

/* The boundary of an outer step of a host-owned DPM-Solver++(2M) loop in ONE pass: lp_boundary_known with the Euler
 * update replaced by sample_dpmpp_2m's:
 *   d   = model_out->combine ? b + (a - b)*cfg : a
 *   out = mask ? y : d                                                  written when out != NULL
 *   x   = ratio*x - em1*out                                             when old_out == NULL (first order)
 *   x   = ratio*x - em1*(c_cur*out - c_old*old_out)                     otherwise (second order)
 *   x   = mask ? rep_noise*noise + rep_y*y : x  (row of next_table)     when next_table != NULL
 * old_out is the previous step's `out`.  The sampler takes the first-order branch on its first step and on the step
 * to sigma = 0: the caller passes old_out == NULL exactly then.  Every operation of the update is the single
 * correctly rounded fp32 operation the eager sampler issues (mul, sub; never contracted), so x equals the un-fused
 * route's bit for bit.  old_out is read only where the update survives (free positions; known positions too when
 * next_table == NULL) and must not overlap x_inout or out.  known may be NULL (dense y / noise / mask).
 *
 * The second-order step of ComfyUI's res_multistep (eta = 0), x = sigma_fn(h)*x + h*(b1*out + b2*old_out), is this
 * launch with ratio = sigma_fn(h), em1 = -h, c_cur = b1 and c_old = -b2, bit for bit: negation is exact, and IEEE 754
 * defines a - b as a + (-b), so c_cur*out - c_old*old_out = b1*out + b2*old_out and ratio*x - em1*s = ratio*x + h*s,
 * each product and sum the same single correctly rounded operation the sampler issues. */
int lp_boundary_multistep(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                          const lp_known* known, float* x_inout, float* out, const float* old_out,
                          const lp_multistep* step, const float* next_table, const lp_dims* dims, lp_stream_t stream);

/* One update of k-diffusion's sample_dpm_2 (DPM-Solver-2, no churn): x_out = x_base + ((x_in - out) / sigma) * dt.
 * The host evaluates sigma and dt with the sampler's own torch expressions on the schedule, on the device the
 * sampler runs on, and reads them back.  Per outer step i with sigma_next > 0:
 *   predictor  sigma = sigma_i,   dt = sigma_mid - sigma_i    x_in = x_base = X,  x_out = X2
 *   corrector  sigma = sigma_mid, dt = sigma_next - sigma_i   x_in = X2, x_base = x_out = X
 * with sigma_mid = exp(lerp(log sigma_i, log sigma_next, 1/2)); the step to sigma_next = 0 is one Euler update,
 * sigma = sigma_i, dt = -sigma_i, x_in = x_base = x_out = X. */
typedef struct lp_midpoint {
  float sigma; /* the sigma the update divides by */
  float dt;    /* the step it multiplies with */
} lp_midpoint;

/* The boundary of a wrapper call of a host-owned DPM-Solver-2 loop in ONE pass: lp_boundary_known with the Euler
 * update replaced by sample_dpm_2's:
 *   d     = model_out->combine ? b + (a - b)*cfg : a
 *   out   = mask ? y : d                                                written when out != NULL
 *   x_out = x_base + ((x_in - out) / sigma) * dt
 *   x_out = mask ? rep_noise*noise + rep_y*y : x_out  (row of next_table)  when next_table != NULL
 * Every operation of the update is the single correctly rounded fp32 operation the eager sampler issues (sub, div,
 * mul, add; never contracted), so x_out equals the un-fused route's bit for bit.  x_in and x_base are read only where
 * the update survives (free positions; known positions too when next_table == NULL), once when they are the same
 * pointer.  Any two of x_in, x_base and x_out are the same buffer or disjoint; out overlaps none of them.  known may
 * be NULL (dense y / noise / mask). */
int lp_boundary_midpoint(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                         const lp_known* known, const float* x_in, const float* x_base, float* x_out, float* out,
                         const lp_midpoint* step, const float* next_table, const lp_dims* dims, lp_stream_t stream);
/* lp_boundary_midpoint with a row-bounded out (see lp_boundary_known_rows). */
int lp_boundary_midpoint_rows(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                              const lp_known* known, const float* x_in, const float* x_base, float* x_out, float* out,
                              int64_t out_rows, const lp_midpoint* step, const float* next_table, const lp_dims* dims,
                              lp_stream_t stream);

/* One outer step of ComfyUI's sample_deis (DEIS, max_order 3, 'tab' mode): x = x + c_cur*d [+ c_prev1*d_{i-1}
 * [+ c_prev2*d_{i-2}]] with d = (x - out) / sigma.  The host takes the coefficients from the sampler's own
 * get_deis_coeff_list (fp32); on a first-order step (the first one, and the step to sigma = 0) c_cur is the fp32
 * difference sigma_next - sigma and the other two are unused. */
typedef struct lp_deis {
  float sigma;   /* the sigma d divides by */
  float c_cur;   /* weight of this step's derivative */
  float c_prev1; /* weight of the previous step's (second- and third-order steps) */
  float c_prev2; /* weight of the one before it (third-order steps) */
} lp_deis;

/* The boundary of an outer step of a host-owned DEIS loop in ONE pass: lp_boundary_known with the Euler update
 * replaced by sample_deis's:
 *   den = model_out->combine ? b + (a - b)*cfg : a
 *   out = mask ? y : den                                                written when out != NULL
 *   d   = (x - out) / sigma
 *   x   = x + c_cur*d                                                   when d_prev1 == NULL (first order)
 *   x   = x + c_cur*d + c_prev1*d_prev1                                 when d_prev2 == NULL (second order)
 *   x   = x + c_cur*d + c_prev1*d_prev1 + c_prev2*d_prev2               otherwise (third order)
 *   d_out = d                                                           written when d_out != NULL
 *   x   = mask ? rep_noise*noise + rep_y*y : x  (row of next_table)     when next_table != NULL
 * d_prev1 and d_prev2 are the d_out of the two previous steps.  Every operation of the update is the single correctly
 * rounded fp32 operation the eager sampler issues (sub, div, mul, add, left to right; never contracted), so x equals
 * the un-fused route's bit for bit.  d_out is written at every position, known ones included: a later step with no
 * next_table (the last step of a window that ends above sigma = 0) updates known positions from it.  d_prev1 and
 * d_prev2 are read only where the update survives (free positions; known positions too when next_table == NULL).
 * d_prev2 needs d_prev1; d_out, d_prev1 and d_prev2 overlap neither each other nor x_inout or out.  known may be NULL
 * (dense y / noise / mask). */
int lp_boundary_deis(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                     const lp_known* known, float* x_inout, float* out, float* d_out, const float* d_prev1,
                     const float* d_prev2, const lp_deis* step, const float* next_table, const lp_dims* dims,
                     lp_stream_t stream);
/* lp_boundary_deis with a row-bounded out (see lp_boundary_known_rows). */
int lp_boundary_deis_rows(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                          const lp_known* known, float* x_inout, float* out, int64_t out_rows, float* d_out,
                          const float* d_prev1, const float* d_prev2, const lp_deis* step, const float* next_table,
                          const lp_dims* dims, lp_stream_t stream);

/* One outer step of ComfyUI's sample_gradient_estimation (ge_gamma, no cfg_pp): the Euler step x = x + d*dt and,
 * from the second step on, the gradient-estimation correction x = x + (gm1*(d - d_prev))*dt, with d = (x - out) / sigma;
 * the step to sigma = 0 is x = out.  The host evaluates sigma and dt with the sampler's own torch expressions on the
 * schedule, on the device the sampler runs on, and reads them back; gm1 is the fp32 value of ge_gamma - 1. */
typedef struct lp_gradient_estimation {
  float sigma; /* sigma_i, the sigma d divides by */
  float dt;    /* sigma_next - sigma_i */
  float gm1;   /* ge_gamma - 1 */
  int final;   /* nonzero on the step to sigma = 0: x = out */
} lp_gradient_estimation;

/* The boundary of an outer step of a host-owned gradient-estimation loop in ONE pass: lp_boundary_known with the Euler
 * update replaced by sample_gradient_estimation's:
 *   den   = model_out->combine ? b + (a - b)*cfg : a
 *   out   = mask ? y : den                                              written when out != NULL
 *   d     = (x - out) / sigma
 *   x     = out                                                         when step->final (the sampler's x = denoised)
 *   x     = x + d*dt                                                    otherwise
 *   x     = x + (gm1*(d - d_prev))*dt                                   when d_prev != NULL (after the line above)
 *   d_out = d                                                           when d_out != NULL, at every position
 *   x     = mask ? rep_noise*noise + rep_y*y : x  (row of next_table)   when next_table != NULL
 * d_prev is the previous step's d_out.  Every operation of the update is the single correctly rounded fp32 operation
 * the eager sampler issues (sub, div, mul, add in its order; never contracted), so x equals the un-fused route's bit
 * for bit.  d_out is written at every position, known ones included: a later step with no next_table (the last step of
 * a window that ends above sigma = 0) updates known positions from it.  d_prev is read only where the update survives
 * (free positions; known positions too when next_table == NULL).  final excludes d_prev; d_out, d_prev, x_inout and
 * out overlap none of each other.  known may be NULL (dense y / noise / mask). */
int lp_boundary_gradient_estimation(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                                    const lp_known* known, float* x_inout, float* out, float* d_out,
                                    const float* d_prev, const lp_gradient_estimation* step, const float* next_table,
                                    const lp_dims* dims, lp_stream_t stream);
/* lp_boundary_gradient_estimation with a row-bounded out (see lp_boundary_known_rows). */
int lp_boundary_gradient_estimation_rows(const lp_heads* model_out, const float* y, const float* noise,
                                         const uint8_t* mask, const lp_known* known, float* x_inout, float* out,
                                         int64_t out_rows, float* d_out, const float* d_prev,
                                         const lp_gradient_estimation* step, const float* next_table,
                                         const lp_dims* dims, lp_stream_t stream);

/* The corrector of k-diffusion's sample_heun (no churn, so sigma_hat = sigma_i): x = x + ((d + d_2) / 2) * dt with
 * d = (x - denoised) / sigma_i from the step's first wrapper call and d_2 = (x_2 - denoised_2) / sigma_next from its
 * second, at x_2 = x + d*dt.  The host evaluates the three scalars with the sampler's own torch expressions on the
 * schedule, on the device the sampler runs on, and reads them back.  Per outer step i with sigma_next > 0:
 *   predictor  lp_boundary_midpoint, sigma = sigma_i, dt,   x_in = x_base = X,  x_out = X2, out = OUT
 *   corrector  lp_boundary_heun,                             x = X, x2 = X2, out_prev = OUT
 * and the step to sigma_next = 0 is lp_boundary_midpoint with x_in = x_base = x_out = X. */
typedef struct lp_heun {
  float sigma;      /* sigma_i, the sigma d divides by */
  float sigma_next; /* sigma_{i+1}, the sigma d_2 divides by */
  float dt;         /* sigma_{i+1} - sigma_i */
} lp_heun;

/* The boundary of the second wrapper call of an outer step of a host-owned Heun loop in ONE pass: lp_boundary_known
 * with the Euler update replaced by sample_heun's corrector:
 *   den = model_out->combine ? b + (a - b)*cfg : a
 *   out = mask ? y : den                                                written when out != NULL
 *   x   = x + ((((x - out_prev) / sigma) + ((x2 - out) / sigma_next)) / 2) * dt
 *   x   = mask ? rep_noise*noise + rep_y*y : x  (row of next_table)     when next_table != NULL
 * out_prev is the first call's out (its pasted denoised latent) and x2 the state the second call ran on.  d is
 * recomputed from x and out_prev with the sampler's operations on the sampler's inputs (x is not written between the
 * two calls), so it has the sampler's bits.  Every operation of the update is the single correctly rounded fp32
 * operation the eager sampler issues (sub, div, add, mul by 1/2, mul, add; never contracted), so x equals the un-fused
 * route's bit for bit.  x, x2 and out_prev are read only where the update survives (free positions; known positions
 * too when next_table == NULL).  x, x2, out_prev and out overlap none of each other.  known may be NULL (dense y /
 * noise / mask). */
int lp_boundary_heun(const lp_heads* model_out, const float* y, const float* noise, const uint8_t* mask,
                     const lp_known* known, float* x, const float* x2, const float* out_prev, float* out,
                     const lp_heun* step, const float* next_table, const lp_dims* dims, lp_stream_t stream);

/* Final denoise of an outer step straight from raw cond / uncond predictions:
 *   out = mask ? y : uncond + (cond - uncond)*cfg ;  if x_inout != NULL: x = x + (x - out)*euler_coef. */
int lp_epilogue_cfg_f32(const float* cond, const float* uncond, float cfg, const float* y, const uint8_t* mask,
                        float* x_inout, float* out, float euler_coef, const lp_dims* dims, lp_stream_t stream);

/* Early-stop statistics (LanPaintEarlyStopper, src/LanPaint/earlystop.py:32-55,238-313):
 *   sums[0] = sum over elements with mask == 0 (the inpaint weight)  of (scale*(a-b))^2
 *   sums[1] = sum over elements with ring != 0 (4-neighbour boundary) of (scale*(a-b))^2
 * i.e. the numerators of _weighted_mse for the inpaint and boundary-ring weights; the denominators are
 * constants of the mask.  ring may be NULL (sums[1] = 0); table may be NULL (scale = 1), otherwise
 * scale = inv_S of the row, which turns a model-space difference into the VP-space one the reference
 * measures on x_t.  ring uses the mask's layout/strides.  sums: 2 doubles on the device, zeroed by the call.
 * Warp-shuffle + one atomicAdd(double) per block per sum. */
int lp_stop_stats_f32(const float* a, const float* b, const uint8_t* mask, const uint8_t* ring,
                      const float* table, const lp_dims* dims, double* sums, lp_stream_t stream);

/* ---- device: utilities (tests, bench) ---------------------------------- */
/* out[i] ~ N(0,1) with the given rng (PHILOX or TORCH; draw0 only). */
int lp_fill_normal_f32(float* out, int64_t n, const lp_rng* rng, lp_stream_t stream);

/* The noise image of a sample call with the bits of ComfyUI's CPU draw.  `comfy.sample.prepare_noise`, which
 * nodes.common_ksampler calls for every LanPaint KSampler node (src/LanPaint/nodes.py:513,589), is
 * `torch.manual_seed(seed); torch.randn(size, generator=..., device="cpu")`: at::mt19937 (one 32-bit output per
 * float, 24 bits kept), torch's normal_fill (Box-Muller over the pairs (j, j+8) of every 16 values; a size that is
 * not a multiple of 16 redraws its last 16) with avx_mathfun.h's cephes log / sincos as the AVX2 build executes them.
 * Writes out[0..n) ~ N(0,1) with exactly those bits (fp32, n >= 16; `out` must have room for n + 16 floats).
 * state_out (optional, 624 words on the device) receives the generator's state array after its last twist and
 * *consumed_out (optional, host) the number of 32-bit outputs drawn, so that the caller can leave the host's CPU
 * generator where ComfyUI's own call would have left it.  One CTA walks the (sequential) generator; the transform
 * is a second, parallel launch. */
int lp_torch_cpu_randn_f32(float* out, int64_t n, uint64_t seed, uint32_t* state_out, int64_t* consumed_out,
                           lp_stream_t stream);

/* Synthetic pointwise two-head denoiser used by bench.py (SURVEY 8d):
 *   h0 = a0*x + b0*tanh(x) + c0 ;  h1 = a1*x + c1     coef = {a0,b0,c0,a1,c1} */
int lp_synth_denoiser_f32(const float* x, float* h0, float* h1, int64_t n, const float* coef5_host,
                          lp_stream_t stream);
/* Same, heads written in `dtype` (a network that computes in bf16 returns bf16 predictions). */
int lp_synth_denoiser(const float* x, void* h0, void* h1, int dtype, int64_t n, const float* coef5_host,
                      lp_stream_t stream);

/* L2 residency for the operands every sub-step re-reads (the clean latent y and the mask: 4 + 1/C of the
 * 28 + 1/C bytes per element).  H100 has 50 MB of L2; pinning y (and the mask that follows it in the same
 * allocation, if any) with a persisting access-policy window turns those reads into L2 hits for the whole
 * job.  lp_l2_persist_set() raises cudaLimitPersistingL2CacheSize to cover `bytes` (clamped to the device
 * maximum; hit_ratio is scaled down accordingly) and installs the window on `stream`: every kernel launched
 * (or captured) on that stream afterwards carries it.  lp_l2_persist_clear() removes the window and resets the
 * persisting lines.  Both are host-side configuration calls, not captured operations. */
int lp_l2_persist_capacity(int device, size_t* max_persisting_bytes, size_t* max_window_bytes);
int lp_l2_persist_set(const void* ptr, size_t bytes, lp_stream_t stream);
int lp_l2_persist_clear(lp_stream_t stream);

/* Writes `bytes` of scratch (> L2) to evict the working set between launches. */
int lp_l2_flush(void* scratch, size_t bytes, lp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LANPAINT_B200_H_ */

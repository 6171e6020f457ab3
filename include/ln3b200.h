/* libln3b200 -- C ABI of the H100-native (sm_90a) LN3Diff generation hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b): every entry point takes a plain-C argument struct
 * of raw device pointers, explicit sizes/strides and enums, plus the CUDA stream as `void*`
 * (a cudaStream_t).  No torch types, no allocation, no retained pointers, no host
 * synchronisation: callers own every buffer (including workspaces).  All entry points return
 * LN3_OK (0) or a negative LN3_E* code; ln3_last_error() returns the thread-local message.
 * There is deliberately no CPU fallback: on a box without an sm_90 GPU every compute call
 * fails with LN3_ECUDA.
 *
 * Each entry point cites the reference code (NIRVANALAN/LN3Diff, paths relative to the
 * reference root) whose device work it replaces.  The reference has no FFI of its own -- it is
 * pure PyTorch -- so the "binding" is the ctypes stub in ln3diff_b200/_lib.py, mirrored for a
 * maintainer in INTEGRATION.md.
 */
#ifndef LN3B200_H_
#define LN3B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LN3_ABI_VERSION 1

#define LN3_OK 0
#define LN3_EINVAL (-1)       /* bad shape / alignment / enum */
#define LN3_ECUDA (-2)        /* CUDA runtime or driver error (includes: no GPU) */
#define LN3_EUNSUPPORTED (-3) /* configuration outside what the kernels implement */

int ln3_abi_version(void);
const char* ln3_last_error(void);
/* Number of kernels this library has launched in this process (for bench.py gpu_launches). */
unsigned long long ln3_launch_count(void);
/* A CUDA graph captured from these entry points re-executes its kernels without passing through
 * the library: callers add the graph's kernel-node count per replay to keep the tally honest. */
void ln3_add_launch_count(unsigned long long n);

/* ------------------------------------------------------------------ GEMM (wgmma + TMA)
 * out = epilogue(A[M,K] . W[N,K]^T): replaces every nn.Linear on the path
 *   dit/dit_models_xformers.py:231-323 (adaLN_modulation, FusedMLP), vit/vision_transformer.py:
 *   106-124 (qkv, proj), ldm/modules/attention.py:245-307 (to_q/k/v/out), dit/dit_decoder.py.
 * A, W bf16 row-major (K contiguous); fp32 accumulation in registers.
 * Epilogue: + bias[N] (fp32, optional) -> activation -> one of
 *   LN3_OUT_BF16       out bf16 [M, ldo]
 *   LN3_OUT_F32        out f32  [M, ldo]
 *   LN3_OUT_RESID_F32  out f32 residual stream updated in place:
 *                      out[m,n] += gate[(m / gate_rows) * gate_ld + n] * val   (gate NULL -> 1)
 *                      and, if out2 != NULL, out2 (bf16 [M, ldo2]) receives the updated row
 *                      (the un-normalised cross-attention query input of TextCondDiTBlock).
 * Constraints: K % 64 == 0, N % 128 == 0, 16-byte aligned pointers and leading dimensions.
 */
enum { LN3_ACT_NONE = 0, LN3_ACT_GELU_ERF = 1, LN3_ACT_GELU_TANH = 2, LN3_ACT_SILU = 3,
       LN3_ACT_QUICK_GELU = 4 /* x * sigmoid(1.702 x): the CLIP towers of the conditioners */ };
enum { LN3_OUT_BF16 = 0, LN3_OUT_F32 = 1, LN3_OUT_RESID_F32 = 2 };

typedef struct ln3_gemm_args {
  const void* A;   /* bf16 [M, lda] */
  const void* W;   /* bf16 [N, ldw] */
  const float* bias;
  void* out;
  void* out2;
  const float* gate;
  int M, N, K;
  long long lda, ldw, ldo, ldo2, gate_ld;
  int gate_rows;
  int act;
  int out_kind;
  /* optional per-head RMSNorm of the first head_norm_nsec column sections (each head_norm_sec_cols
   * wide, heads of 64 columns) before the bf16 store: y = x * rsqrt(mean_64(x^2) + eps) * w[sec][i].
   * This is `q, k = self.q_norm(q), self.k_norm(k)` (qk_norm=True, RMSNorm(64, eps 1e-5):
   * vit/vision_transformer.py:81-82,116; ldm/modules/attention.py:264-265,294) fused into the
   * projection GEMM.  head_norm_w: fp32 [head_norm_nsec, 64] or NULL.  LN3_OUT_BF16 only. */
  const float* head_norm_w;
  int head_norm_nsec;
  int head_norm_sec_cols;
  float head_norm_eps;
  /* reserved scratch (the kernel needs none: ln3_gemm_workspace_bytes() returns 0); ignored. */
  void* workspace;
  size_t workspace_bytes;
} ln3_gemm_args;

size_t ln3_gemm_workspace_bytes(void);

int ln3_gemm_bf16(const ln3_gemm_args* args, void* stream);

/* ------------------------------------------------------------------ attention (wgmma)
 * out[b, i, h*hd:(h+1)*hd] = softmax(q_h k_h^T * scale) v_h, no mask: replaces
 * xformers.ops.memory_efficient_attention at vit/vision_transformer.py:114-118 (packed qkv of
 * MemEffAttention), ldm/modules/attention.py:279-307 (cross-attention, incl. its three
 * permute+contiguous copies) and the DiT2 decoder attention (dit/dit_decoder.py).
 * q/k/v/out are bf16; head h of row i of batch b lives at ptr + b*bs + i*ld + h*hd, so a packed
 * (B, N, 3, H, hd) qkv buffer is addressed as q = base, k = base + H*hd, v = base + 2*H*hd with
 * ld = 3*H*hd.  Lq and Lkv are arbitrary (tails are zero-filled by TMA and masked).
 * head_dim (hd) is 64 (DiT-S/B/L, the PixArt denoisers, the DiT2 VAE, CLIP) or 72 (DiT-XL/2: 1152 / 16 heads);
 * any other value returns LN3_EUNSUPPORTED.  At head_dim 72 a second K/V source (k2/v2) returns
 * LN3_EUNSUPPORTED; causal works at both widths.  `scale` is the caller's (head_dim ** -0.5 in every model).
 */
typedef struct ln3_fmha_args {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  int B, H, Lq, Lkv, head_dim;
  long long q_ld, q_bs, k_ld, k_bs, v_ld, v_bs, o_ld, o_bs; /* elements */
  float scale;
  /* optional second K/V source appended after the first along the sequence (any Lkv / Lkv2): the step-invariant DINO tokens the I23D blocks concatenate to the latent
   * tokens for self-attention (dit/dit_models_xformers.py:522-530) -- their K/V are cached per
   * prompt and never copied.  k2/v2 NULL -> unused. */
  const void* k2;
  const void* v2;
  int Lkv2;
  long long k2_ld, k2_bs, v2_ld, v2_bs;
  /* causal != 0: key j is visible to query i only when j <= i (the CLIP text tower of FrozenCLIPEmbedder,
   * sgm/modules/encoders/modules.py:347-408 -> transformers CLIPTextModel's causal mask); not with k2/v2. */
  int causal;
} ln3_fmha_args;

int ln3_fmha_fwd(const ln3_fmha_args* args, void* stream);

/* ------------------------------------------------------------------ norm + modulate (adaLN)
 * out_bf16[r, :] = norm(x[r, :]) * (1 + scale[g(r), :] (+ scale_tab)) + shift[g(r), :] (+ shift_tab)
 * with g(r) = r / mod_rows.  Replaces `modulate(self.norm1(x), shift, scale)` /
 * `t2i_modulate(...)` (dit/dit_models_xformers.py:47-53, 285-294, 518-530) and `modulate2` with
 * per-token operands (dit/dit_decoder.py:15-17; mod_rows = 1), producing the bf16 GEMM operand.
 *   norm = LN3_NORM_LAYER: LayerNorm without affine, biased variance, eps (1e-6 on the path)
 *          LN3_NORM_RMS  : x * rsqrt(mean(x^2) + eps) * weight        (dit/norm.py:27-40)
 *          LN3_NORM_NONE : identity (plain fp32 -> bf16 cast, optional activation LN3_ACT_*)
 * shift/scale NULL -> no modulation.  D must be a multiple of 128 and <= 2048.
 * Alignment (LN3_EINVAL otherwise): x, out, shift, scale, shift_tab, scale_tab, weight, resid, resid_gate,
 * resid_out_gate and resid_bcast 16-byte aligned; ldx, ldo, mod_ld, resid_ld, resid_gate_ld and
 * resid_out_gate_ld multiples of 4, resid_bcast_ld a multiple of 8.
 */
enum { LN3_NORM_NONE = 0, LN3_NORM_LAYER = 1, LN3_NORM_RMS = 2 };

/* OSG decoder arithmetic of the renderer / point queries */
enum { LN3_MLP_FP32 = 0, LN3_MLP_TF32 = 1 };

typedef struct ln3_norm_modulate_args {
  const float* x;     /* [rows, ldx]; updated in place when `resid` is given */
  void* out;          /* bf16 [rows, ldo] (NULL allowed with `resid`) */
  const float* shift; /* [groups, mod_ld] or NULL */
  const float* scale;
  const float* shift_tab; /* [D] or NULL: PixArt scale_shift_table rows */
  const float* scale_tab;
  const float* weight;    /* RMS weight [D] or NULL */
  int rows, D;
  long long ldx, ldo, mod_ld;
  int mod_rows;
  int norm;
  int act;            /* applied last (only with LN3_NORM_NONE) */
  float eps;
  /* optional fused residual update executed first, in place on x:
   *   x[r,:] += resid_gate[(r / resid_gate_rows), :] * resid[r,:]      (gate NULL -> 1)
   * i.e. the `x = x + gate * f(...)` of the DiT blocks (dit/dit_models_xformers.py:289-294,
   * 311-321) applied to the bf16 output of the preceding projection GEMM, so the residual stream is
   * read and written once, coalesced, by the kernel that normalises it anyway.  out may be NULL
   * (residual update only). */
  const void* resid;       /* bf16 [rows, resid_ld] or NULL */
  const float* resid_gate; /* fp32 [groups, resid_gate_ld] or NULL */
  long long resid_ld, resid_gate_ld;
  int resid_gate_rows;
  /* optional: rows outside [resid_row_begin, resid_row_end) take their residual from a per-group row
   *   resid_bcast[(r / resid_bcast_rows), :]   (bf16, row pitch resid_bcast_ld)
   * instead of resid[r,:] -- the cross-attention output of samples whose context tokens are all
   * identical (the zero-embedding unconditional half of classifier-free guidance,
   * sgm/modules/diffusionmodules/guiders.py:33-44 with force_uc_zero_embeddings): softmax over identical
   * keys is uniform, so the attention output is the one value row for every query.  NULL -> unused. */
  const void* resid_bcast;
  long long resid_bcast_ld;
  int resid_bcast_rows, resid_row_begin, resid_row_end;
  /* optional, with resid_bcast: the rows OUTSIDE [resid_row_begin, resid_row_end) additionally add their own
   * row of `resid` under a second gate,
   *   x[r,:] += resid_out_gate[(r / resid_out_gate_rows), :] * resid[r,:] + resid_bcast[...]
   * -- for those samples the preceding `x += gate_msa * attn` (dit/dit_models_xformers.py:311-312) has not been
   * applied yet: the pass that applies it exists only to produce the bf16 cross-attention query input, which the
   * closed-form samples do not need, so their self-attention and cross-attention residuals are applied together
   * here and the in-between pass covers the attended rows only.  NULL -> unused. */
  const float* resid_out_gate;
  long long resid_out_gate_ld;
  int resid_out_gate_rows;
} ln3_norm_modulate_args;

int ln3_norm_modulate(const ln3_norm_modulate_args* args, void* stream);

/* ------------------------------------------------------------------ timestep embedding
 * out_bf16[b, 0:128] = cos(t_b f_i), out[b, 128:256] = sin(t_b f_i), f_i = exp(-ln(1e4) i/128):
 * TimestepEmbedder.timestep_embedding (dit/dit_models_xformers.py:97-121), dim 256.
 */
int ln3_timestep_embedding(const float* t, int B, void* out_bf16, void* stream);

/* ------------------------------------------------------------------ patch embed (roll-out)
 * tokens[b, n*L + l, :] = Conv2d(k=s=2)(x[b, c*3+n, :, :])[l] + bias + pos_embed[n*L + l, :]
 * i.e. rearrange 'b (c n) h w -> (b n) c h w' + timm PatchEmbed + pos_embed
 * (dit/dit_trilatent.py:93-99).  x fp32 (B, 3*Cin, S, S) optionally pre-scaled per sample by
 * in_scale[b] (the denoiser's c_in, sgm/modules/diffusionmodules/denoiser.py:34-42);
 * weight fp32 (D, Cin, 2, 2); tokens fp32 (B, 3*(S/2)^2, D).  S even, 1 <= Cin <= 16.  Cin == 4 with D % 4 == 0
 * takes the vectorised kernel only when weight, bias, pos_embed and tokens are 16-byte aligned.
 */
typedef struct ln3_patch_embed_args {
  const float* x;
  const float* in_scale; /* [B] or NULL */
  const float* weight;
  const float* bias;
  const float* pos_embed; /* [3*L, D] or NULL */
  float* tokens;
  int B, Cin, S, D;
} ln3_patch_embed_args;

int ln3_patch_embed(const ln3_patch_embed_args* args, void* stream);

/* ------------------------------------------------------------------ multi-view conditioner: Plücker patchify
 * The bf16 GEMM A-operand of the 9-channel 14x14 patch embedding of FrozenDinov2ImageEmbedderMVPlucker
 * (sgm/modules/encoders/modules.py:955-1013): gen_rays + get_plucker_ray per view, the RGB | Plücker cat, the
 * cast to bf16 and the im2col of Conv2d(9, D, 14, stride 14), in one pass.
 *   image fp32 [N, 3, 224, 224]  pre-processed views (resized and normalised)
 *   cams  fp32 [N, 25]           16 row-major cam2world + 9 intrinsics (fx, fy, cx, cy = c[16], c[20], c[18], c[21])
 *   out   bf16 [N*256, ldo]      row n*256 + py*16 + px, column ch*196 + ky*14 + kx (Conv2d.weight.reshape(D, -1)
 *                                order), channels [r, g, b, (o x d).xyz, d.xyz]; columns [1764, ldo) are zeroed so
 *                                that K = 1792 = 28*64 feeds ln3_gemm_bf16 as it is.
 * Per pixel (x, y): u = (x + 0.5)/224, v = (y + 0.5)/224, dir = normalize(((u - cx)/fx, (v - cy)/fy, 1)),
 * d = R dir, o = t.  Rounding is the reference's under the engine's bf16 autocast: dir and norm in fp32;
 * `c2w[:3,:3] @ dirs` is an autocast matmul (bf16 R and dir, fp32 sum, bf16 d); `torch.cross(o, d)` is promoted
 * to fp32 with fp32 o; the final `.to(bf16)` rounds all nine channels once.  Every fp32 step is individually
 * rounded (no FMA contraction).  Checked on an H100 against torch running the reference's ops under CUDA bf16
 * autocast: 99.998% of the ray elements are bit-identical; the others are pixels where cuBLAS's bf16 batched matmul
 * rounded a partial sum of R . dir (|delta d| <= 2^-8 sum_j |R_ij dir_j|), which this kernel sums once in fp32.
 * LN3_EINVAL unless ldo >= 1764, ldo % 8 == 0 and image, cams and out are 16-byte aligned.
 */
typedef struct ln3_plucker_patchify_args {
  const float* image;
  const float* cams;
  void* out;
  int N;
  long long ldo;
} ln3_plucker_patchify_args;

int ln3_plucker_patchify(const ln3_plucker_patchify_args* args, void* stream);

/* ------------------------------------------------------------------ final layer + unpatchify
 * FinalLayer / T2IFinalLayer (dit/dit_models_xformers.py:61-84, 655-678): LayerNorm(no affine,
 * eps 1e-6) -> modulate(shift, scale (+ tables)) -> Linear(D -> 4*Cout) -> unpatchify ->
 * '(b n) c h w -> b (c n) h w' (dit/dit_trilatent.py:130-140), fp32 contiguous output
 * (B, 3*Cout, S, S).  shift/scale are [B, mod_ld] rows.
 * LN3_EINVAL unless: S even, Cout > 0, D a multiple of 128 and <= 2048, mod_ld a multiple of 4, shift_tab and
 * scale_tab both given or both NULL, and x, shift, scale, the tables and weight 16-byte aligned.
 */
typedef struct ln3_final_layer_args {
  const float* x; /* tokens [B, 3*L, D] */
  const float* shift;
  const float* scale;
  const float* shift_tab;
  const float* scale_tab;
  const float* weight; /* [4*Cout, D] fp32 */
  const float* bias;   /* [4*Cout] */
  float* out;
  int B, S, D, Cout;
  long long mod_ld;
} ln3_final_layer_args;

int ln3_final_layer(const ln3_final_layer_args* args, void* stream);

/* ------------------------------------------------------------------ fused sampler update
 * x_out[b] = a[b] * x[b] + w0[b] * m0[b] + w1[b] * m1[b] + s[b] * noise[b]   (per-sample scalars)
 * One launch per step covering (SURVEY.md section 8a row S*):
 *   Euler-EDM + EpsScaling + VanillaCFG  sgm/modules/diffusionmodules/sampling.py:93-107,
 *       denoiser.py:25-42, guiders.py:24-31, sampling_utils.py:34-35  (m0 = uncond, m1 = cond)
 *   DDPM p_sample (eps/x0/v, fixed variance)  guided_diffusion/gaussian_diffusion.py:273-546
 *   flow-matching Euler + CFG              transport/integrators.py:101-120, dit/dit_i23d.py:155-168
 * coef is [B, 4] = (a, w0, w1, s); m1 / noise may be NULL when their weight is unused.
 * n_per_sample % 4 == 0; x, m0, m1, noise, coef and x_out 16-byte aligned (LN3_EINVAL otherwise).
 */
typedef struct ln3_sampler_update_args {
  const float* x;
  const float* m0;
  const float* m1;
  const float* noise;
  const float* coef;
  float* x_out;
  int B;
  long long n_per_sample;
} ln3_sampler_update_args;

int ln3_sampler_affine_update(const ln3_sampler_update_args* args, void* stream);

/* ------------------------------------------------------------------ fused sampler step (sgm sampler family)
 * The elementwise tail of one denoiser evaluation of every sgm EDM-family sampler, per element of sample b
 * (all scalars per sample, coef row b = (k0, k1, k2, a, b, c, h0, h1, h2, s, 0, 0), [B, 12] fp32):
 *   e = k0 * x_eval + k1 * net_u + k2 * net_c        the guided denoised D, or the derivative d
 *   v = a * x + b * x_eval + c * e + h0 * hist[0] + h1 * hist[1] + h2 * hist[2] + s * noise
 *   x_out[b] = v;  eval_out[b] = eval_out[B + b] = v (both halves of the next 2B CFG input);  hist_out[b] = e
 * evaluated left to right as one fmaf chain.  net_u / net_c are the network's uncond / cond output halves
 * (EpsScaling: D = x_eval - sigma_q * net); net_c is NULL for IdentityGuider; a NULL hist[j] or noise drops its
 * term; a NULL output is not written.  Covers:
 *   VanillaCFG / IdentityGuider + DiscreteDenoiser(EpsScaling)   guiders.py:24-42, denoiser.py:25-42,
 *       denoiser_scaling.py:29-37
 *   EulerAncestralSampler    sampling.py:133-170,237-244 (ancestral Euler + noise), sampling_utils.py:22-35
 *   HeunEDMSampler           sampling.py:93-107,218-234 (predictor writes x_euler + d, corrector averages)
 *   DPMPP2SAncestralSampler  sampling.py:247-284, sampling_utils.py:38-43 (midpoint evaluation, mult1..4)
 *   DPMPP2MSampler           sampling.py:287-362 (previous guided D in hist[0])
 *   LinearMultistepSampler   sampling.py:173-208, sampling_utils.py:7-19 (up to 3 past derivatives)
 * n_per_sample % 4 == 0; every non-NULL pointer 16-byte aligned; x, x_eval, net_u and coef non-NULL; at least one
 * output.  x_eval, net_*, hist[j], noise and x_out hold B rows, eval_out 2B rows.  No output may overlap another
 * output or an input, except x_out == x and eval_out == x_eval (same start: the element is read before it is
 * written by the same thread).  LN3_EINVAL otherwise, before any CUDA call.
 */
typedef struct ln3_sampler_step_args {
  const float* x;
  const float* x_eval;
  const float* net_u;
  const float* net_c;
  const float* hist[3];
  const float* noise;
  const float* coef;
  float* x_out;
  float* eval_out;
  float* hist_out;
  int B;
  long long n_per_sample;
} ln3_sampler_step_args;

int ln3_sampler_step(const ln3_sampler_step_args* args, void* stream);

/* ------------------------------------------------------------------ flow-matching SDE step
 * The elementwise tail of one drift evaluation of the transport's SDE samplers (transport/integrators.py:9-75,
 * transport/transport.py:246-372, path.py:18-110: Euler-Maruyama and Heun on the Linear path with velocity
 * prediction) around a CFG denoiser.  The state has 2R rows of n elements: rows [0, R) are the conditional half,
 * [R, 2R) the unconditional half, R = P * N condition-major (P conditions of N samples).  The two halves diverge
 * (each row draws its own noise), but both move under the same guided velocity.  For state row r, j = r mod R:
 *   v   = f[R+j] + s * (f[j] - f[R+j])       guided velocity (f: the forward output, conditional rows first)
 *   sc  = (t * v - y[r]) / var               score at the evaluated input y (var = sigma_t^2 + t sigma_t)
 *   d   = v + D * sc (LN3_SDE_DRIFT) | v (LN3_SDE_VELOCITY) | sc (LN3_SDE_SCORE)
 *   o(k) = k[0] * x[r] + k[1] * y[r] + k[2] * d + k[3] * hist[r] + k[4] * w[noise_row(r)]
 *   x_out[r] = o(cx);  y_out[r] = o(cy);  hist_out[r] = d
 * v, sc and d are rounded as the reference's separate fp32 tensor ops (no contraction); o is one fmaf chain, left
 * to right.  Each output has its own coefficients, so the state can be written without the noise term while the
 * next forward's input gets it.  noise_row(r) = (r < R ? 0 : N) + (j mod N): w is one (2N, n) draw whose rows
 * [0, N) serve the conditional half and [N, 2N) the unconditional half of every condition, as P sequential
 * samplers seeded alike would draw.  A NULL x, hist or noise drops its term; a NULL output is not written.
 * R >= 0; n % 4 == 0; y and f non-NULL; at least one output; mode one of LN3_SDE_*; with noise, 0 < N <= R and
 * R % N == 0; every non-NULL pointer 16-byte aligned.  x, y, f, hist and every output hold 2R rows, noise 2N.
 * No output may overlap another output or an input, except x_out == x and y_out == y (same start: the element is
 * read before it is written by the same thread).  LN3_EINVAL otherwise, before any CUDA call.
 */
enum { LN3_SDE_DRIFT = 0, LN3_SDE_VELOCITY = 1, LN3_SDE_SCORE = 2 };

typedef struct ln3_flow_sde_step_args {
  const float* x;       /* [2R, n] state (optional) */
  const float* y;       /* [2R, n] the evaluated input */
  const float* f;       /* [2R, n] forward output at y */
  const float* hist;    /* [2R, n] optional */
  const float* noise;   /* [2N, n] optional */
  float* x_out;
  float* y_out;
  float* hist_out;
  float cx[5];          /* x_out: (a, b, c, h, sigma) */
  float cy[5];          /* y_out: (a, b, c, h, sigma) */
  float cfg_scale, t, var, diffusion;
  int mode;
  int R, N;
  long long n;
} ln3_flow_sde_step_args;

int ln3_flow_sde_step(const ln3_flow_sde_step_args* args, void* stream);

/* ------------------------------------------------------------------ grouped adaptive dopri5
 * The per-attempt arithmetic of the adaptive Dormand-Prince 5(4) solver that `sample_ode`'s default runs
 * (transport/transport.py:374-421 -> transport/integrators.py:101-120 -> torchdiffeq odeint(method='dopri5')),
 * restated in transport/dopri5.py, for G independent problems in one batch.  Row r of the fp32 state
 * [B, n_per_sample] belongs to group row_group[r]; each group has its own error norm, step size, accept / reject,
 * counters and end, held in the caller-owned device array `state` [G] of ln3_ode_group.  Times and steps are
 * float64, as the host solver keeps them; the forward's per-row time is fp32.  No host synchronisation: the caller
 * reads `status` back (asynchronously) to learn when every group has finished.
 *   ln3_ode_stage(stage 1..6): y_stage = y + sum_j beta[stage-1][j] * dt_g * k_j (k_0 = f0, k_j = k[j-1]) and
 *       t_rows[r] = fp32(t_g + alpha[stage-1] * dt_g); stage 0 is the initial-step probe y_stage = y + h0_g * f0,
 *       t_rows = t_g + h0_g.  Rows of groups whose status is not LN3_ODE_RUNNING are not written.
 *   ln3_ode_initial_step(phase 0): per group d0 = rms(y / s), d1 = rms(f0 / s), s = atol + rtol |y|, h0 (dt = h0);
 *       (phase 1, after one forward of the stage-0 probe into k[0]): d2 = rms((k[0] - f0) / s) / h0, h1 and
 *       dt = min(100 h0, h1) (order 4, Hairer-Norsett-Wanner II.4); nfe = 2.
 *   ln3_ode_step: after the six stage forwards (k[0..5]; y_stage holds the 5th-order solution y1):
 *       ratio = rms(err / (atol + rtol max(|y|, |y1|))), err = dt * sum_j c_err[j] k_j; accept iff ratio <= 1;
 *       dt' = dt * min(ifactor, max(safety / ratio^(1/5), accepted ? 1 : dfactor)), dt * ifactor when ratio == 0;
 *       on accept y <- y1, f0 <- k[5] (FSAL), and when t reaches t_end the quartic dense output at t_end is written
 *       to out and the group is done.  Then the checks of the next attempt: accepted + rejected >= max_num_steps
 *       gives LN3_ODE_EMAXSTEPS, t + dt == t gives LN3_ODE_EUNDERFLOW (the group is frozen; the kernels never trap).
 * Reductions are deterministic: every row is cut into fixed chunks of 1024 elements whose squares are summed in a
 * fixed order into `workspace` (float64), and each group sums its rows' partials in row, then chunk, order -- a
 * group's result does not depend on the other groups in the batch.
 * LN3_EINVAL unless B, G > 0, n_per_sample > 0 and % 4 == 0, every row_group_host entry in [0, G) with every group
 * non-empty, workspace_bytes >= ln3_ode_workspace_bytes(B, n_per_sample), the state, row map, time and the buffers
 * an entry point reads or writes non-NULL, and y, f0, k[], y_stage and out 16-byte aligned.
 */
enum { LN3_ODE_RUNNING = 0, LN3_ODE_DONE = 1, LN3_ODE_EMAXSTEPS = -1, LN3_ODE_EUNDERFLOW = -2 };

typedef struct ln3_ode_group {
  double t;        /* time reached (end of the last accepted step) */
  double dt;       /* size of the next attempt (h0 between the two initial-step phases) */
  double t_prev;   /* start of the last accepted step */
  double dt_step;  /* size of the last attempt */
  double ratio;    /* error ratio of the last attempt */
  double aux;      /* initial-step scratch (d1) */
  int nfe, accepted, rejected;
  int status;      /* LN3_ODE_RUNNING, LN3_ODE_DONE or a negative LN3_ODE_E* code */
  int event;       /* last attempt: 0 rejected / not run, 1 accepted, 2 accepted and reached t_end */
  int reserved;
} ln3_ode_group;

typedef struct ln3_ode_args {
  float* y;                     /* [B, n] state, committed on accept */
  float* f0;                    /* [B, n] derivative at y (FSAL) */
  const float* k[6];            /* [B, n] stage derivatives of the current attempt */
  float* y_stage;               /* [B, n] forward input written by ln3_ode_stage */
  float* t_rows;                /* [B] fp32 forward time written by ln3_ode_stage */
  float* out;                   /* [B, n] dense output at t_end, written once per group */
  const int* row_group;         /* device int32 [B] */
  const int* row_group_host;    /* host copy of row_group, validated on every call */
  ln3_ode_group* state;         /* device [G] */
  void* workspace;              /* device, ln3_ode_workspace_bytes(B, n_per_sample) */
  size_t workspace_bytes;
  int B, G;
  long long n_per_sample;
  double t_end, rtol, atol, safety, ifactor, dfactor;
  int max_num_steps;
} ln3_ode_args;

size_t ln3_ode_workspace_bytes(int B, long long n_per_sample);
int ln3_ode_stage(const ln3_ode_args* args, int stage, void* stream);
int ln3_ode_initial_step(const ln3_ode_args* args, int phase, void* stream);
int ln3_ode_step(const ln3_ode_args* args, void* stream);

/* ------------------------------------------------------------------ grouped adaptive Runge-Kutta
 * The ln3_ode_* arithmetic above for torchdiffeq's other explicit adaptive Runge-Kutta methods (torchdiffeq 0.2.3
 * bosh3.py, fehlberg2.py, adaptive_heun.py; restated in transport/rk.py), selected by `method`:
 *   LN3_ODE_DOPRI5         6 stages, order 5, FSAL   (ln3_ode_stage / _initial_step / _step are this method)
 *   LN3_ODE_BOSH3          3 stages, order 3, FSAL   (Bogacki-Shampine 3(2))
 *   LN3_ODE_FEHLBERG2      2 stages, order 2         (Runge-Kutta-Fehlberg 2(1))
 *   LN3_ODE_ADAPTIVE_HEUN  1 stage,  order 2         (Heun-Euler 2(1))
 * With S = ln3_ode_stages(method): stages 1..S take beta[stage-1] and alpha[stage-1] of the method's tableau; the
 * step reads k[0 .. S-1]; nfe grows by S per attempt; the controller and the initial step use 1/order in place of
 * 1/5; the dense output uses the method's mid weights and f1 = k[S-1].  For a tableau that is not FSAL (c_sol is not
 * the last beta row with a trailing 0), ln3_ode_rk_step first overwrites y_stage with y1 = y + dt sum_j c_sol[j] k_j
 * (one more launch), and still commits f0 <- k[S-1], the derivative at the last stage's input, as torchdiffeq does.
 * Everything else, and every rule on the arguments, is that of the dopri5 entry points.  An unknown method returns
 * LN3_EUNSUPPORTED (ln3_ode_stages returns it too), a stage outside 0..S LN3_EINVAL.
 */
enum { LN3_ODE_DOPRI5 = 0, LN3_ODE_BOSH3 = 1, LN3_ODE_FEHLBERG2 = 2, LN3_ODE_ADAPTIVE_HEUN = 3 };

int ln3_ode_stages(int method);
int ln3_ode_rk_stage(const ln3_ode_args* args, int method, int stage, void* stream);
int ln3_ode_rk_initial_step(const ln3_ode_args* args, int method, int phase, void* stream);
int ln3_ode_rk_step(const ln3_ode_args* args, int method, void* stream);

/* ------------------------------------------------------------------ tri-plane volumetric renderer
 * ln3_render_views: the whole of ImportanceRenderer.forward (nsr/volumetric_rendering/renderer.py:
 * 133-307) for the Objaverse presets (nsr/script_util.py:761-797, 838-870): 'auto' ray limits against the
 * box (math_utils.py:124-190, renderer.py:145-155), S stratified + S importance samples per ray,
 * tri-plane bilinear gather (renderer.py:55-104), in-box filter (:381-405), OSGDecoder
 * (nsr/triplane.py:339-375, FullyConnectedLayer gains nsr/networks_stylegan2.py:141-145),
 * MipRayMarcher2 (ray_marcher.py:26-68), sample_importance / sample_pdf (:479-552) and
 * unify_samples (:422-435), fused into one persistent warp-per-ray kernel.
 *
 *   planes_cl    fp32 [n_obj, 3, H, W, 32] channels-last (ln3_planes_to_channels_last)
 *   view_obj     int32 [V] object of each view, or NULL -> view v uses object v / views_per_obj
 *   ray_o, ray_d fp32 [V, M, 3]           (ln3_generate_rays, or caller supplied)
 *   S, S_importance  equal, 64 (objaverse_tuneray_aug_resolution_64_64_auto) or 96 (..._96_96_auto, the
 *                preset of the DiT2-L/2 VAE); any other count is LN3_EUNSUPPORTED
 *   noise_*      fp32 [V, M, S] uniform [0,1): the tensors the reference draws with
 *                torch.rand_like (renderer.py:464) and torch.rand (renderer.py:530)
 *   w1,b1,w2,b2  raw OSGDecoder parameters (64,32), (64), (4,64), (4) -- gains applied inside
 *   rgb          fp32 [V, 3, M]  ('feature_samples' permuted: image_raw when reshaped to H x W)
 *   depth        fp32 [V, 1, M]   weights fp32 [V, 1, M]
 * group_size consecutive views share the reference's per-call global reductions (min/max of the
 * valid ray starts, depth clamp range): 1 when the reference renders one view per call
 * (nsr/train_util_diffusion.py:292-302), N for a batched Triplane.forward.
 * workspace: ln3_render_workspace_bytes(V, M, group_size) bytes of device memory.
 * dbg_* (optional, tests only): per-sample in-box masks [V*M,2S] (coarse ++ fine), searchsorted
 * indices [V*M,S], sort permutation [V*M,2S], fine depths [V*M,S].
 */
typedef struct ln3_render_args {
  const float* planes_cl;
  const int* view_obj;
  const float* ray_o;
  const float* ray_d;
  const float* noise_coarse;
  const float* noise_fine;
  const float* w1;
  const float* b1;
  const float* w2;
  const float* b2;
  float* rgb;
  float* depth;
  float* weights;
  void* workspace;
  size_t workspace_bytes;
  unsigned char* dbg_inbox;
  int* dbg_inds;
  int* dbg_order;
  float* dbg_zfine;
  int V, M, H, W, C, S, S_importance, hidden_dim, decoder_output_dim;
  int group_size, views_per_obj, white_back;
  int mlp_precision; /* LN3_MLP_FP32 (exact, SIMT) or LN3_MLP_TF32 (mma.sync tensor cores, fp32 accumulate) */
  double box_warp, bbox_min, bbox_max;
  /* optional: the M rays of a view are the pixels of an image of this width, m = y * image_w + x (RaySampler
   * order, ray_sampler.py:180-195).  When width and height are multiples of 4 the kernel walks 4x4 pixel tiles
   * (16 co-resident warps march through neighbouring texels in step: L1 reuse); 0 = plain ray order. */
  int image_w;
} ln3_render_args;

size_t ln3_render_workspace_bytes(int V, int M, int group_size);
/* The schedule ln3_render_views takes for M rays per view and args->image_w: the image width when the kernel
 * walks 4x4 pixel tiles, 0 when it walks the rays in plain order (16 consecutive rays per work item). */
int ln3_render_tile_width(int M, int image_w);
int ln3_render_views(const ln3_render_args* args, void* stream);

/* ------------------------------------------------------------------ tri-plane point queries
 * ImportanceRenderer._run_model (nsr/volumetric_rendering/renderer.py:310-322) as driven by
 * forward_points / triplane_decode_grid (vit/vit_triplane.py:2009-2120) for mesh extraction:
 * sample_from_planes (bilinear, zeros padding, box_warp) + OSGDecoder at arbitrary points; no in-box
 * filter, no compositing.  sigma[n_obj][P] is the raw density logit, rgb[n_obj][P][3] the sigmoid
 * colour.  points == NULL -> the kernel generates the reference's grid itself (torch.linspace per axis
 * over [aabb_min, aabb_max], meshgrid 'ij'), P = grid_size^3: no 85 MB coordinate tensor, no
 * 2^16-point chunking, no empty_cache() between chunks.
 */
typedef struct ln3_query_points_args {
  const float* planes_cl; /* [n_obj][3][H][W][C] channels-last */
  const float* points;    /* [n_obj][P][3] or NULL (grid mode) */
  const float* w1;
  const float* b1;
  const float* w2;
  const float* b2;
  float* sigma;
  float* rgb;
  long long P;
  int n_obj, C, H, W, hidden_dim, decoder_output_dim, grid_size;
  int mlp_precision; /* LN3_MLP_FP32 or LN3_MLP_TF32 */
  float aabb_min_x, aabb_min_y, aabb_min_z, aabb_max_x, aabb_max_y, aabb_max_z;
  double box_warp;
} ln3_query_points_args;

int ln3_query_points(const ln3_query_points_args* args, void* stream);

/* RaySampler.forward (nsr/volumetric_rendering/ray_sampler.py:180-257): cams fp32 [V, 25]
 * (16 cam2world row-major + 9 intrinsics) -> ray_o, ray_d fp32 [V, res*res, 3], ray m = y*res + x. */
int ln3_generate_rays(const float* cams, int V, int res, float* ray_o, float* ray_d, void* stream);

/* (n_obj, 3*32, H, W) fp32 tri-plane as the VAE decoder emits it (vit/vit_triplane.py:1964,
 * channel = plane*32 + c) -> channels-last [n_obj, 3, H, W, 32] for the renderer's gathers. */
int ln3_planes_to_channels_last(const float* planes, int n_obj, int C, int H, int W, float* out,
                                void* stream);

/* ------------------------------------------------------------------ mesh extraction: marching cubes
 * Replaces the CPU `mcubes.marching_cubes(grid_out['sigma'] as (G,G,G) numpy, mesh_thres)` call of the mesh
 * export (nsr/train_util_diffusion.py:221-223; PyMCubes is an un-vendored third-party package) that follows
 * the G^3 point query (ln3_query_points).  grid fp32 [nx][ny][nz] (z fastest), exactly the array the reference
 * hands to mcubes.  Output is an indexed mesh like PyMCubes':
 *   vertices fp32 [n_vertices][3] = (i, j, k) index coordinates of the iso crossing on a lattice edge
 *            (linear interpolation, `value <= iso` classifies a corner), times scale[] plus offset[] per axis
 *            (scale 1 / offset 0 = mcubes; 2/(G-1)*0.45 and -0.45 fold the reference's :225-226 rescale in);
 *            ordered by (owning lattice point's linear index, axis)
 *   faces    int32 [n_faces][3] vertex indices, ordered by the cell's linear index; winding of the classic
 *            case table (normal towards the `<= iso` side), case tables generated by tools/gen_mc_tables.py.
 * Two calls because the sizes are data dependent: `_count` classifies and scans (totals[0] = n_vertices,
 * totals[1] = n_faces, device ints the caller reads back), `_emit` writes at most max_vertices / max_faces
 * entries.  workspace: ln3_marching_cubes_workspace_bytes(nx, ny, nz) bytes, 256-byte aligned, the SAME buffer
 * (contents preserved) for both calls. */
typedef struct ln3_marching_cubes_args {
  const float* grid;
  void* workspace;
  size_t workspace_bytes;
  int* totals;      /* device int[2] */
  float* vertices;  /* emit only */
  int* faces;       /* emit only */
  int nx, ny, nz;
  int max_vertices, max_faces;
  float iso;
  float scale[3];
  float offset[3];
} ln3_marching_cubes_args;

size_t ln3_marching_cubes_workspace_bytes(int nx, int ny, int nz);
int ln3_marching_cubes_count(const ln3_marching_cubes_args* args, void* stream);
int ln3_marching_cubes_emit(const ln3_marching_cubes_args* args, void* stream);

/* ------------------------------------------------------------------ frame sink
 * TrainLoopDiffusionWithRec.render_video_given_triplane's per-view host loop
 * (nsr/train_util_diffusion.py:292-376): `.cpu()` + numpy + matplotlib per view, replaced by one device
 * pass over all views so that one batched D2H copy (or the NCCL all-gather of frames) moves uint8.
 *   image  fp32 [N,3,H,W] in [-1,1] ('image_raw')
 *   depth  fp32 [N,1,H,W] ('image_depth') or NULL
 *   out    u8 [N, H, Wout, 3] (HWC video frames), Wout = W, or 2W with depth: [image | colour-mapped depth]
 * Arithmetic as the reference: byte = uint8(clip(v * 127.5 + 127.5, 0, 255)) (truncation), evaluated in float64
 * for the video frame with depth (the cat with the float64 colormap output promotes it, :340-345,366-368) and in
 * float32 (two rounded operations) for the image-only frame (the per-view image dump, :350-353);
 * depth -> (d - min_view) / (max_view - min_view) in fp32, colormap index min(trunc(x * 256), 255), the
 * byte table `lut` u8 [256,3] = uint8(clip((cmap_rgb * 2 - 1) * 127.5 + 127.5, 0, 255)) of the 256-entry
 * colormap (plt.cm.viridis in the reference); max == min gives the colormap's "bad" colour (0,0,0).
 * workspace: 2*N floats (per-view min / max).  W % 4 == 0. */
typedef struct ln3_pack_frames_args {
  const float* image;
  const float* depth;
  const unsigned char* lut;
  unsigned char* out;
  float* workspace;
  int N, H, W;
} ln3_pack_frames_args;

int ln3_pack_frames(const ln3_pack_frames_args* args, void* stream);

/* ------------------------------------------------------------------ VAE decoder: conv tail (NHWC fp32)
 * The reference's superresolution['conv_sr'] = ldm Decoder (ldm/modules/diffusionmodules/model.py:
 * 625-731) and PatchEmbedTriplane (vit/vit_triplane.py:58-108).  Activations are NHWC so the DiT2
 * token stream feeds conv_in directly and conv_out writes the renderer's channels-last tri-plane.
 *
 * ln3_conv_nhwc: out = conv(ksize in {1,3}, stride 1, pad ksize/2)(f(up(x))) + bias (+ residual)
 *   f = identity, or the fused GroupNorm-apply (+ swish): v*in_scale[n,c] + in_shift[n,c]
 *       (model.py:46-52 nonlinearity / Normalize; scale/shift from ln3_groupnorm_stats)
 *   up = identity or nearest 2x (Upsample, model.py:54-69): x is then [N, H/2, W/2, Cin]
 *   w is the Conv2d weight repacked to [ksize*ksize, Cin, Cout].  H, W are the OUTPUT dims.
 *   LN3_EUNSUPPORTED for ksize not 1 or 3.  LN3_EINVAL for a precision other than LN3_MLP_FP32 / LN3_MLP_TF32
 *   (TF32 applies to ksize 3; ksize 1 always runs fp32), N < 0, non-positive H, W, Cin or Cout, upsample with odd
 *   H or W, only one of in_scale / in_shift, or a NULL x, w or out -- checked before N == 0 returns without a launch.
 * ln3_conv_cout_tile: the output channels per CTA (32 or 64) ln3_conv_nhwc takes for these dims: 32 when
 *   Cout < 64 or when 64-channel CTAs would give fewer than two per SM of the current device; 0 for a
 *   non-positive argument.
 * ln3_groupnorm_stats: torch.nn.GroupNorm(G, C, eps) statistics of x [N, HW, C] folded with the
 *   affine parameters into per-(image, channel) scale / shift [N, C].  N <= 0 returns without a launch;
 *   otherwise LN3_EINVAL for non-positive G, C or HW, C % G != 0, C / G > 256 or a NULL pointer.
 * ln3_attn_single_head: MemoryEfficientAttnBlock core (model.py:209-272): softmax(q k^T/sqrt(C)) v,
 *   q/k/v/out fp32 [N, L, C], one head of width C (128 in conv_sr).  N <= 0 returns without a launch;
 *   otherwise LN3_EINVAL for L <= 0 or a NULL pointer, LN3_EUNSUPPORTED for C not 32, 64 or 128.
 * ln3_patch_embed_triplane: Conv2d(3*Cz -> 3*E, k=s=2, groups=3) + the reference's
 *   (B,3E,h,w)->(B,E,3,h,w)->(B,3hw,E) reshape; x fp32 [B, 3*Cz, S, S] is pre-multiplied by in_mul
 *   (triplane_scaling_divider, nsr/train_util_diffusion.py:188); optional bf16 SiLU copy of the
 *   tokens (the adaLN operand of every DiT2 block, dit/dit_decoder.py:29-31).  B <= 0 returns without a
 *   launch; otherwise LN3_EINVAL for Cz outside 1..16, odd or non-positive S, E <= 0 or a NULL x, w or tokens
 *   (bias and silu_bf16 may be NULL).
 */
typedef struct ln3_conv_args {
  const float* x;
  const float* w;
  const float* bias;
  const float* in_scale;
  const float* in_shift;
  const float* residual;
  float* out;
  int N, H, W, Cin, Cout, ksize, upsample, in_swish;
  int precision; /* LN3_MLP_FP32 (exact SIMT) or LN3_MLP_TF32 (3x3 only: mma.sync tensor cores, fp32 accumulate) */
} ln3_conv_args;

int ln3_conv_nhwc(const ln3_conv_args* args, void* stream);
int ln3_conv_cout_tile(int N, int H, int W, int Cout);
int ln3_groupnorm_stats(const float* x, const float* gamma, const float* beta, int N, int HW, int C,
                        int G, float eps, float* scale, float* shift, void* stream);
int ln3_attn_single_head(const float* q, const float* k, const float* v, float* out, int N, int L,
                         int C, void* stream);
int ln3_patch_embed_triplane(const float* x, const float* w, const float* bias, int B, int Cz, int S,
                             int E, float in_mul, float* tokens, void* silu_bf16, void* stream);

/* ------------------------------------------------------------------ VAE encoder (NHWC fp32)
 * The stage-1 encoder MVEncoder (ldm/modules/diffusionmodules/model.py:459-577) runs on ln3_conv_nhwc,
 * ln3_groupnorm_stats, ln3_gemm_bf16, ln3_fmha_fwd and ln3_norm_modulate plus the two entry points below.
 *
 * ln3_downsample_nhwc: Downsample (model.py:72-91): out = conv3x3(F.pad(x, (0,1,0,1)), stride 2, no padding) + bias.
 *   Here H, W are the INPUT dims and must be even; x [N, H, W, Cin], out [N, H/2, W/2, Cout], w repacked to
 *   [9, Cin, Cout] as for ln3_conv_nhwc.  precision LN3_MLP_FP32 (exact SIMT) or LN3_MLP_TF32 (mma.sync, fp32
 *   accumulate).  LN3_EINVAL for odd H or W, ksize != 3, upsample, in_scale / in_shift, residual, another precision,
 *   non-positive sizes or a NULL x, w or out.
 *
 * ln3_vae_posterior: vae_encode + DiagonalGaussianDistribution(soft_clamp=True) + sample() / mode() of the AE
 *   decoder (vit/vit_triplane.py:912-933, 1152-1199; utils/torch_utils/distributions/distributions.py:29-113):
 *     moments fp32 [B, S, S, 24]  the fused encoder output, NHWC
 *     w fp32 [24, 8], bias [24]   quant_conv = Conv2d(24, 24, 1, groups=3)
 *     noise fp32 [B, 12, S, S]    the standard-normal draw of sample(), or NULL for mode(): z = mean
 *     mean, logvar, z fp32 [B, 12, S, S] (the layout of latent_normalized_2Ddiffusion)
 *   with q = quant_conv(moments), mean[:, j] = q[:, j], lv = q[:, 12 + j] (the reference's reshape to (B, 8, 3, H, W)
 *   and chunk), logvar = 20 tanh(lv / 20), z = mean + exp(0.5 logvar) * noise.  Each fp32 step after the 8-term dot
 *   product is rounded on its own, as torch evaluates it.  LN3_EINVAL for B < 0, S <= 0 or a NULL pointer other than
 *   noise.
 */
int ln3_downsample_nhwc(const ln3_conv_args* args, void* stream);

typedef struct ln3_vae_posterior_args {
  const float* moments;
  const float* w;
  const float* bias;
  const float* noise;
  float* mean;
  float* logvar;
  float* z;
  int B, S;
} ln3_vae_posterior_args;

int ln3_vae_posterior(const ln3_vae_posterior_args* args, void* stream);

/* ln3_view_mean_nhwc: the view pooling of MVEncoderGSDynamicInp (ldm/modules/diffusionmodules/model.py:611-623),
 * feat.mean(keepdim=True, dim=0) over each object's F consecutive views:
 *   x fp32 [B*F, S, S, C] NHWC -> out fp32 [B, S, S, C],
 *   out[b, i] = (((x[b*F, i] + x[b*F + 1, i]) + ...) + x[b*F + F-1, i]) / F
 * summed over the views in order in fp32, each addition rounded to nearest, then one IEEE division by F.
 * LN3_EINVAL for F <= 0, B < 0, S <= 0, C <= 0 or a NULL x / out (checked before B == 0 returns without a
 * launch).  out must not overlap x. */
int ln3_view_mean_nhwc(const float* x, float* out, int B, int F, int S, int C, void* stream);

/* ------------------------------------------------------------------ FP8 (e4m3) denoiser GEMMs
 * An opt-in operating point for the qkv / fc1 / fc2 GEMMs of the DiT blocks.  Its results are NOT held to the
 * reference's parity tolerance: fp8 operands move the outputs by far more than bf16 rounding does.
 *
 * Number format.  Codes are e4m3 with the encoding and the +-448 saturation of torch.float8_e4m3fn.
 *   Activations: 1 x 128 block scales.  A is e4m3 [M, K] with fp32 a_scale[M, K/128]; block (m, kb) covers
 *     columns [128 kb, 128 kb + 128) of row m and is quantised as
 *       s = fp32(absmax / 448)            (IEEE division; an all-zero block has s = 0 and zero codes)
 *       q = e4m3_rn_satfinite(fp32(x / s))
 *     so x ~ q * s.  ln3_quantize_fp8_rows, ln3_norm_modulate_fp8 and the LN3_OUT_FP8 epilogue all write this.
 *   Weights: per output channel.  W is e4m3 [N, K] with fp32 w_scale[N] (quantised once, off the hot path, with
 *     torch's float8_e4m3fn cast of W / w_scale, w_scale = absmax of the row / 448).
 *
 * ln3_gemm_fp8: out = epilogue(w_scale[n] * sum_kb a_scale[m, kb] * P(m, n, kb)),  P = sum_{k in kb} q_a q_w.
 *   Each 128-deep partial P comes out of the tensor core's fp8 MMA (whose internal accumulation is narrower
 *   than fp32) in an accumulator of its own and is added, scaled by a_scale, into a separate fp32 accumulator:
 *   acc = fmaf(a_scale[m, kb], P, acc).  Then y = fmaf(acc, w_scale[n], bias[n]) and one of
 *     LN3_OUT_BF16 with LN3_ACT_NONE   bf16 [M, ldo], optionally with the per-head RMSNorm of ln3_gemm_args
 *                                      (head_norm_*, same semantics) before the store
 *     LN3_OUT_FP8 with LN3_ACT_NONE or LN3_ACT_GELU_ERF (the polynomial of the bf16 GEMM's fc1 epilogue)
 *                                      e4m3 [M, ldo] with block scales out_scale[M, N/128] (pitch out_scale_ld),
 *                                      the operand format above, so fc1 writes fc2's A directly.
 *   Deterministic: no split-K, no atomics; each output sees the same instructions in the same order whatever
 *   the grid.  LN3_EINVAL unless M > 0, K % 128 == 0, N % 128 == 0, A, W, out 16-byte aligned, lda, ldw and the
 *   output row pitch in bytes multiples of 16, a_scale and w_scale given, a_scale_ld >= K/128, bias 16-byte
 *   aligned, and with LN3_OUT_FP8 out_scale given with out_scale_ld >= N/128.  LN3_EUNSUPPORTED for any other
 *   output kind / activation pairing and for head_norm outside LN3_OUT_BF16.  There is no bf16 fallback.
 *
 * ln3_norm_modulate_fp8: ln3_norm_modulate (`base`: the same residual update, norm and modulation, the same
 *   residual-stream arithmetic bit for bit) writing the e4m3 + block-scale format instead of bf16.  base.out must
 *   be NULL (base.ldo is ignored).  LN3_EINVAL for the checks of ln3_norm_modulate plus out / out_scale NULL or
 *   misaligned (out 16 bytes, ldo % 16), out_scale_ld < D/128; LN3_EUNSUPPORTED unless D % 256 == 0, D <= 1536,
 *   base.ldx % 8 == 0, x 32-byte aligned and (with resid) resid_ld % 8 == 0.
 *
 * ln3_quantize_fp8_rows: x (fp32, or bf16 when x_bf16 != 0) [rows, ldx] -> out e4m3 [rows, ldo] + out_scale
 *   [rows, out_scale_ld].  rows <= 0 returns without a launch; otherwise LN3_EINVAL for a NULL pointer, D not a
 *   positive multiple of 128, ldx < D, ldo < D or out_scale_ld < D/128, ldx % 4 (fp32) / % 8 (bf16), ldo % 16 or
 *   x / out not 16-byte aligned.
 */
enum { LN3_OUT_FP8 = 3 };

typedef struct ln3_gemm_fp8_args {
  const void* A;         /* e4m3 [M, lda] */
  const float* a_scale;  /* [M, a_scale_ld] */
  const void* W;         /* e4m3 [N, ldw] */
  const float* w_scale;  /* [N] */
  const float* bias;     /* [N] or NULL */
  void* out;             /* bf16 or e4m3 [M, ldo] */
  float* out_scale;      /* LN3_OUT_FP8: [M, out_scale_ld] */
  int M, N, K;
  long long lda, ldw, ldo, a_scale_ld, out_scale_ld;
  int act;
  int out_kind;
  const float* head_norm_w;
  int head_norm_nsec;
  int head_norm_sec_cols;
  float head_norm_eps;
  /* reserved scratch (ln3_gemm_fp8_workspace_bytes() returns 0); ignored. */
  void* workspace;
  size_t workspace_bytes;
} ln3_gemm_fp8_args;

size_t ln3_gemm_fp8_workspace_bytes(void);
int ln3_gemm_fp8(const ln3_gemm_fp8_args* args, void* stream);

typedef struct ln3_norm_modulate_fp8_args {
  ln3_norm_modulate_args base;
  void* out;         /* e4m3 [rows, ldo] */
  float* out_scale;  /* [rows, out_scale_ld] */
  long long ldo, out_scale_ld;
} ln3_norm_modulate_fp8_args;

int ln3_norm_modulate_fp8(const ln3_norm_modulate_fp8_args* args, void* stream);
int ln3_quantize_fp8_rows(const void* x, int x_bf16, long long ldx, int rows, int D, void* out, long long ldo,
                          float* out_scale, long long out_scale_ld, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LN3B200_H_ */

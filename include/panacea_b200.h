/*
 * panacea_b200 — C ABI of the H100-native Panacea denoising hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b). The reference is pure Python with no FFI of its own; the
 * interface this library stands behind is the `nn.Module.forward` surface of
 *   sgm/modules/diffusionmodules/wrappers.py:37-70     OpenAIWrapperControlLDM3D.forward
 *   sgm/modules/diffusionmodules/controlmodel.py:86-202 ControlNet3D / ControlledUNetModel3D.forward
 *   sgm/modules/diffusionmodules/openaimodel.py:499-542 ResBlock3D._forward
 *   sgm/modules/attention.py:407-610,229-291,1064-1134  view / text / temporal attention, STT
 *   sgm/modules/diffusionmodules/sampling.py:85-365     EDM (Euler with churn, Heun), ancestral (Euler-a,
 *                                                       DPM++ 2S-a), DPM++ 2M and LMS solver steps
 * and every entry point below names the reference call site it replaces. The Python host
 * (panacea_b200/sgm/...) mirrors those classes and binds these symbols with ctypes (INTEGRATION.md).
 *
 * Conventions
 *  - plain pointers + sizes only; all tensor pointers are DEVICE pointers owned by the caller;
 *  - activations are channels-last: fp32 residual stream [frames, H, Wtot, C], bf16 MMA operands;
 *    frame index = b*T + t (t fastest), Wtot = 6 views side by side (view-major along W);
 *  - `stream` is a cudaStream_t passed as void*; every call is asynchronous on it and allocation-free
 *    (CUDA-graph capturable); a handle-free design: no hidden device state except memoised TMA maps;
 *  - return 0 on success, negative pn_status otherwise; message via pn_last_error() (thread-local);
 *  - there is NO CPU fallback anywhere: without a CUDA device every compute entry point fails.
 */
#ifndef PANACEA_B200_H
#define PANACEA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Changes when an existing entry point or struct changes or goes; an added entry point leaves it, since every caller
 * of the previous surface still links and behaves the same. */
#define PN_ABI_VERSION 4

enum pn_status { PN_STATUS_OK = 0, PN_STATUS_INVALID = -1, PN_STATUS_CUDA = -2, PN_STATUS_UNSUPPORTED = -3 };

/* How a producer writes the A operand of the GEMM that follows it ("operand_mode" arguments below).
 *  PN_OPERAND_BF16   bf16 [rows, C]                   — the fast path (bf16 products, fp32 accumulation);
 *  PN_OPERAND_SPLIT3 bf16 [rows, 3C] = [hi | lo | hi] — parity mode: hi = bf16(v), lo = bf16(v - hi); against weights
 *                    packed [W_hi | W_hi | W_lo] per tap the same pn_gemm kernel yields fp32-class products
 *                    (hi W_hi + lo W_hi + hi W_lo), which is how the reference's fp32 math (wrappers.py:37-70 on CPU)
 *                    is matched to rtol 1e-3 / atol 1e-4;
 *  PN_OPERAND_F32    fp32 [rows, C]                   — input of a CUDA-core consumer in parity mode;
 *  PN_OPERAND_SPLIT3_B bf16 [rows, 3C] = [hi | hi | lo] — the WEIGHT form (the layout ops.split3 packs weights in), made
 *                    on the device for a GEMM whose B factor is an activation (the VAE mid-block attention's k and v).
 *                    Only pn_cast_operand accepts it; every other entry point with an operand_mode rejects it. */
enum pn_operand_mode { PN_OPERAND_BF16 = 0, PN_OPERAND_SPLIT3 = 1, PN_OPERAND_F32 = 2, PN_OPERAND_SPLIT3_B = 3 };

const char* pn_last_error(void);
int pn_abi_version(void);

/* ------------------------------------------------------------------------------------------------
 * pn_gemm — wgmma GEMM / implicit-GEMM convolution (sm_90a, TMA + mbarrier pipeline).
 * Replaces: nn.Linear (attention.py:94,113,220-226; openaimodel.py:939-941), nn.Conv2d 3x3 stride 1 over
 * the 6-view panorama (openaimodel.py:413,455-462,125), nn.Conv1d k=3 over frames (openaimodel.py:418,
 * 468-476), 1x1 skip / zero convs (openaimodel.py:486; controlmodel.py:81-84).
 *   out[row, n] = epi( sum_{th,tw,c} A[nb, y+th-taps_h/2, x+tw-taps_w/2, c] * B[n, (th*taps_w+tw)*C + c] )
 * with zero padding outside [0,H)x[0,W) and row = (nb*H + y)*W + x.
 * epi: + bias[n] + rowvec[(row / rows_per_group) % n_groups, n]; GEGLU (columns in blocks of 32 = 16 value
 * columns then the 16 gate columns of the same outputs -> N/2 outputs, out = value * gelu_erf(gate), attention.py:91-99); + residual[row, n] + residual2[row, n] (fp32); store fp32 or bf16.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pn_gemm_args {
  const void* A;          /* bf16 [NB, H, W, C] with element strides below (C contiguous) */
  const void* B;          /* bf16 [N, taps_h*taps_w*C], K contiguous */
  void* out;              /* fp32 or bf16 [NB*H*W, ldo] */
  const float* bias;      /* [N] or NULL */
  const float* rowvec;    /* [n_groups, N] or NULL */
  const void* residual;   /* fp32 (or bf16 when residual_bf16) [NB*H*W, ldr] or NULL (may alias out when same dtype) */
  const float* residual2; /* second fp32 addend [NB*H*W, ldr2] or NULL (fp32 output only) */
  int64_t NB, H, W, C;
  int64_t a_stride_w, a_stride_h, a_stride_n; /* elements */
  int64_t ldo, ldr, ldr2;
  int64_t rowvec_ld;      /* row stride of rowvec in elements (0 = N) */
  int32_t N;
  int32_t taps_h, taps_w;
  int32_t rows_per_group, n_groups;
  int32_t out_bf16;
  int32_t geglu;
  int32_t residual_bf16;  /* the residual is bf16 (bf16 output only): the transformer blocks' bf16 token stream */
  /* LayerNorm folded into the GEMMs around the bf16 token stream (attention.py:699-701 + :726-747, norm1/2/3):
   * ln_stats_out — this GEMM (bf16 out, no GEGLU) also writes, per output row, pn_gemm_ln_parts(N) partial
   *   (sum, sum of squares) pairs: float [rows][parts][2]. With BN = 160 if N % 160 == 0 else 128, part 2 * t + h
   *   sums columns [t * BN + h * BN/2, t * BN + (h + 1) * BN/2) (half h of column tile t), taken from the fp32 values
   *   before their bf16 rounding (only the per-row totals are meaningful to a consumer);
   * ln_stats_in / ln_parts_in / ln_colsum / ln_eps — (1x1, bf16 out, no GEGLU) A is the UN-normalised stream, B = W diag(gamma); the epilogue
   *   finishes the LayerNorm: out = rstd_m (acc - mean_m s_n) + bias_n with s_n = ln_colsum[n] = sum_k B[n,k] and the
   *   caller's bias_n = sum_k beta_k W[n,k] (+ the layer's own bias); mean/rstd over the C = K channels of row m. */
  const float* ln_stats_in;
  const float* ln_colsum;
  float* ln_stats_out;
  int32_t ln_parts_in;
  float ln_eps;
} pn_gemm_args;

int pn_gemm(const pn_gemm_args* args, void* stream);
int pn_gemm_ln_parts(int N);

/* ------------------------------------------------------------------------------------------------
 * Attention. Each entry point serves both precision modes through its operand_mode:
 *  PN_OPERAND_BF16                    q/k/v/out bf16, tensor-core kernels (fp32 softmax), strides in bf16 elements;
 *  PN_OPERAND_SPLIT3 / PN_OPERAND_F32 parity mode: q/k/v fp32 (strides in floats, multiples of 4), fp32 products,
 *                                     softmax and accumulation on CUDA cores; `out` is the dense operand of the to_out
 *                                     GEMM [tokens, heads*head_dim] in that mode, so out_ld must equal heads*head_dim.
 * Any other mode returns PN_STATUS_INVALID.
 *
 * pn_attention — flash attention over view-tiled tokens (head_dim 64 or 80; bf16: wgmma).
 * Replaces: xformers.ops.memory_efficient_attention inside MemoryEfficientIntraViewAttention.forward
 * (attention.py:407-489) and MemoryEfficientInterViewAttentionTwo.forward (attention.py:518-610), and
 * F.scaled_dot_product_attention inside CrossAttention.forward for the 77-token text context
 * (attention.py:229-291). Query tokens are a grid [F, H, V, W] (frame, row, view, column) with token
 * stride q_ld; key/value tokens a grid [F / kv_frame_div, Hk, Vk, Wk] with stride kv_ld. Query view v
 * attends the key views kv_views[v][0 .. kv_view_count[v]) (all rows/columns of those views):
 *   intra-view : kv_views[v] = {v};   cross-view : the reference's table {5,1},{0,2},{1,3},{2,4},{3,5},{4};
 *   text       : V = Vk = 1, W = tokens per batch element, Wk = 77, kv_views[0] = {0}.
 * out[token, head*head_dim + d] = softmax(q k^T * scale) v, token stride out_ld.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pn_attn_args {
  const void* q;   /* channel 0 of head 0 of the first query token */
  const void* k;   /* likewise for keys (may point into the same fused qkv buffer) */
  const void* v;
  void* out;
  int64_t q_ld, kv_ld, out_ld;
  int64_t F, H, V, W;
  int64_t Hk, Vk, Wk;
  int32_t kv_frame_div;
  int32_t heads, head_dim;
  int32_t kv_views[8][2];
  int32_t kv_view_count[8];
  float scale;
} pn_attn_args;

int pn_attention(const pn_attn_args* args, int operand_mode, void* stream);

/* Temporal self-attention over T <= 16 frames per pixel (attention.py:1116-1125 -> :229-291, context=None).
 * q/k/v [batch, T, pixels, ld], out [batch, T, pixels, out_ld]; head_dim 64 or 80. bf16: one (batch, pixel, head)
 * sequence per warp (warp-level bf16 MMAs, fp32 softmax), ld and out_ld multiples of 8. */
int pn_attention_temporal(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t T,
                          int64_t pixels, int32_t heads, int32_t head_dim, int64_t ld, int64_t out_ld, float scale,
                          int operand_mode, void* stream);

/* Causal self-attention of the OpenCLIP text transformer (reference sgm/modules/encoders/modules.py:618-629, each
 * resblock's nn.MultiheadAttention with attn_mask = -inf above the diagonal: token i attends keys j <= i).
 * q/k/v [batch, L, ld] (e.g. three base pointers into the fused in_proj output), out [batch, L, out_ld]; L <= 128,
 * head_dim 64. bf16: one CTA per (batch, head), warp-level bf16 MMAs, fp32 softmax, ld and out_ld multiples of 8. */
int pn_attention_causal(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t L, int32_t heads,
                        int32_t head_dim, int64_t ld, int64_t out_ld, float scale, int operand_mode, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Normalisation (fp32 residual stream in, bf16 MMA operand out)
 * ---------------------------------------------------------------------------------------------- */
/* GroupNorm(32, C) over (C/32, all pixels of a frame) [+ SiLU]: util.py:276-283 (eps 1e-5, ResBlock3D
 * in/out_layers, openaimodel.py:413,455) and attention.py:129-132 (eps 1e-6, STT norm*). The statistics span
 * all six views of the panorama. raw_bf16 (optional) receives a plain bf16 cast of x (input of the 1x1 skip
 * convolution, openaimodel.py:486). workspace: pn_groupnorm_workspace_floats(...) floats. */
int64_t pn_groupnorm_workspace_floats(int64_t frames, int64_t pixels, int64_t channels);
/* How many pixel ranges pn_groupnorm_silu splits each frame's statistics into for a call of this shape. Each frame's
 * result depends on the frame count only through this number, so calls over subsets of the frames that give the same
 * value reproduce one call over all of them bit for bit (the VAE's frame chunking checks it). */
int64_t pn_groupnorm_ctas_per_frame(int64_t frames, int64_t pixels, int64_t channels);
int pn_groupnorm_silu(const float* x, const float* gamma, const float* beta, void* y, void* raw,
                      float* workspace, int64_t frames, int64_t pixels, int64_t channels, float eps, int act_silu,
                      int operand_mode, void* stream);
/* GroupNorm(32, C) over (C/32, T) per pixel [+ SiLU] on x[batch, T, pixels, C]: the reference applies
 * nn.GroupNorm to the "(b h w) c t" rearrangement (openaimodel.py:509-512, 534-537). */
int pn_groupnorm_pixel_silu(const float* x, const float* gamma, const float* beta, void* y, int64_t batch,
                            int64_t frames_per_seq, int64_t pixels, int64_t channels, float eps, int act_silu,
                            int operand_mode, void* stream);
/* nn.LayerNorm(C) per token, eps 1e-5 (attention.py:699-701). x: fp32, or bf16 (x_is_bf16: the bf16 token stream the
 * fast path keeps inside a transformer block). */
int pn_layernorm(const void* x, int x_is_bf16, const float* gamma, const float* beta, void* y, int64_t rows,
                 int64_t channels, float eps, int operand_mode, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Convolutions that cannot feed a 64-wide wgmma K block, layout and sampler helpers
 * ---------------------------------------------------------------------------------------------- */
/* Direct 3x3 conv, pad 1, stride 1|2, channels-last (stem openaimodel.py:977, head :1251, BEV hint stem
 * controlmodel.py:43-59). w_packed fp32 [9][Cin][Cout_pad]; y = act(conv + bias) + addend. */
int pn_conv3x3_direct(const void* x, int x_is_bf16, const float* w_packed, const float* bias, const float* addend,
                      float* y_f32, void* y_bf16, int64_t frames, int64_t H, int64_t W, int64_t Cin, int64_t Cout,
                      int64_t Cout_pad, int stride, int act_silu, void* stream);
/* im2col for the stride-2 Downsample conv: fp32 [F,H,W,C] -> operand [F*Ho*Wo, 9 taps x C] (each tap is one operand
 * row of C channels: 9*C bf16, or 9*3C in split3 mode). pad = 1: Conv2d(3, stride 2, padding 1) of the UNet
 * (openaimodel.py:187); pad = 0: the VAE encoder's F.pad(x, (0,1,0,1)) + Conv2d(3, stride 2, padding 0) (model.py:98-113). */
int pn_im2col3x3_s2(const float* x, void* out, int64_t frames, int64_t H, int64_t W, int64_t C, int pad, int operand_mode,
                    void* stream);
/* F.interpolate(scale_factor=2, mode="nearest") of Upsample (openaimodel.py:133-140), fp32 -> operand. */
int pn_upsample2x(const float* x, void* y, int64_t frames, int64_t H, int64_t W, int64_t C, int operand_mode, void* stream);
/* out = cat([h, skip + ctrl], channel) — decoder skip join (controlmodel.py:193-195); ctrl may be NULL. */
int pn_concat_add(const float* h, const float* skip, const float* ctrl, float* out, int64_t rows, int64_t C1,
                  int64_t C2, void* stream);
int pn_add_inplace(float* x, const float* y, int64_t n, void* stream);      /* h += control.pop() (controlmodel.py:192) */
/* fp32 [rows, C] -> operand: bf16, split3 A form [hi | lo | hi] or split3 weight form [hi | hi | lo] (operand_mode 0, 1, 3). */
int pn_cast_operand(const float* x, void* y, int64_t rows, int64_t C, int operand_mode, void* stream);
/* Parity-mode GEGLU (attention.py:97-99, exact erf GELU) on the fp32 output of the ff.net.0 GEMM whose columns are in
 * pn_gemm's GEGLU packing (blocks of 32 = 16 value + 16 gate columns): in fp32 [rows, 2*inner] -> operand [rows, inner]. */
int pn_geglu_operand(const float* in, void* y, int64_t rows, int64_t inner, int operand_mode, void* stream);
/* y = 0.5 x (1 + erf(x / sqrt 2)): the exact GELU of the OpenCLIP text MLP (reference modules.py:618-629, resblock
 * mlp = c_fc, GELU, c_proj), fp32 [rows, C] (the c_fc output) -> operand of the c_proj GEMM. */
int pn_gelu_operand(const float* x, void* y, int64_t rows, int64_t C, int operand_mode, void* stream);
/* out[b, l, :] = table[tokens[b, l], :] + pos[l, :], fp32 (reference modules.py:610-611, token_embedding +
 * positional_embedding). The caller range-checks the int64 ids against vocab; an id outside [0, vocab) gives NaN. */
int pn_token_embedding(const int64_t* tokens, const float* table, const float* pos, float* out, int64_t batch, int64_t L,
                       int64_t vocab, int64_t width, void* stream);
/* in[batch, A, first B of in_ld columns] -> out[batch, B, ld] at column offset off: NCHW <-> channels-last at the module
 * boundary (also performs the channel concat of wrappers.py:41, and drops the padding columns of the out-head GEMM). */
int pn_transpose_f32(const float* in, float* out, int64_t batch, int64_t A, int64_t B, int64_t in_ld, int64_t out_ld,
                     int64_t out_off, void* stream);
/* util.py:224-248 timestep_embedding (cos | sin halves). freqs: optional fp32 [dim/2] frequency table computed by the
 * host with the reference's expression (bit-identical arguments t*f); NULL = computed in the kernel. */
int pn_timestep_embedding(const int64_t* t, float* out, int64_t n, int64_t dim, const float* freqs, void* stream);
/* y = act_out(W act_in(x) + b) for M <= 32 rows: time_embed MLP and per-block emb_layers
 * (openaimodel.py:936-943, 439-445). */
int pn_linear_small(const float* x, const void* W, int w_is_f32, const float* bias, float* y, int64_t M, int64_t N,
                    int64_t K, int64_t ldy, int silu_in, int silu_out, void* stream);
/* out[r, :] = softmax(scale * in[r, :]), fp32 scores -> the A operand of the O = P v GEMM. With two pn_gemm calls around it
 * this is the single-head attention of the VAE mid block (reference sgm/modules/diffusionmodules/model.py:374-414,
 * head_dim = C). operand_mode PN_OPERAND_BF16 (out bf16 [rows, N]) or PN_OPERAND_SPLIT3 (out bf16 [rows, 3N] =
 * [hi | lo | hi], parity mode). ld_out counts bf16 elements (>= 3N for split3). N <= 51,200 (the row is staged in shared
 * memory), N % 4 == 0. */
int pn_softmax_rows_operand(const float* in, void* out, int64_t rows, int64_t N, int64_t ld_in, int64_t ld_out, float scale,
                            int operand_mode, void* stream);
/* Content fingerprint of a device buffer (two order-independent 64-bit sums over its 32-bit words) -> out2[2] on the
 * device. The wrapper keys its step-invariant conditioning cache (BEV hint stem, text K/V; wrappers.py:37-70 recomputes
 * them every step) on the CONTENT of c["cond_feat"] / c["crossattn"]: addresses are recycled by the allocator. */
int pn_fingerprint(const void* x, int64_t nbytes, uint64_t* out2, void* stream);
/* out[c*n + i] = x[i] * s for c < copies (prepare_sampling_loop x *= sqrt(1+sigma0^2), CFG batch doubling). */
int pn_scale_dup(const float* x, float* out, int64_t n, float s, int copies, void* stream);

/* ------------------------------------------------------------------------------------------------
 * pn_sampler_step — one launch after every network evaluation of a sampler (sampling.py:85-365,
 * sampling_utils.py:12-48), fp32, grid-stride, allocation-free. Per element, in the reference's fp32 order:
 *   xe  = x_eval ? x_eval : x                         the point the network was evaluated at
 *   D_h = net_is_denoised ? net_h : net_h * (-sigma_q) + xe      (denoiser.py:22-28, EpsScaling: c_skip 1, c_out -sigma_q)
 *   D   = halves == 2 ? D_0 + cfg_scale (D_1 - D_0) : D_0       (VanillaCFG, unconditional half first; IdentityGuider)
 *   o   = the mode's update (pn_sampler_mode)
 *   o  += (xi * noise_scale) * noise_amp              when noise_amp != 0; xi = noise[e], or, with noise == NULL, the
 *                                                     standard normal Philox4x32-10(key seed, counter (e / 4, draw)) +
 *                                                     Box-Muller: a function of (seed, draw, e) only
 *   out = o (out == NULL: x, in place);  x_in_next[h * n + e] = o * c_in_next for h < halves (when non-NULL).
 * hist is a ring of n-element slots: the Heun predictor's d, the LMS d_{i-j}, the DPM++ 2M D_{i-1}. A slot may be read
 * and written by the same launch (element-wise, read first).
 * ---------------------------------------------------------------------------------------------- */
enum pn_sampler_mode {
  /* o = xe + dt * d, d = (xe - D) / sigma; hist[hist_write] = d. EulerEDMSampler and EDMSampler with churn
   * (sampling.py:96-110, sigma = sigma_hat, dt = sigma_next - sigma_hat), HeunEDMSampler's predictor (out = stage
   * buffer) and its last step, EulerAncestralSampler (:240-247, dt = sigma_down - sigma, noise_amp = sigma_up) and
   * DPMPP2SAncestralSampler when sigma_down = 0 (:270-272). */
  PN_SAMPLER_EULER = 0,
  /* o = x + ((hist[hist_read[0]] + d') / 2) * dt, d' = (xe - D) / sigma: HeunEDMSampler's corrector (:229-235),
   * evaluated at the predictor xe = stage, sigma = sigma_next. */
  PN_SAMPLER_HEUN = 1,
  /* o = x + (coef[0] d + sum_{j>=1} coef[j] hist[hist_read[j-1]]), d = (xe - D) / sigma, hist[hist_write] = d:
   * LinearMultistepSampler (:194-209), coefficients from linear_multistep_coeff (sampling_utils.py:12-24). */
  PN_SAMPLER_LMS = 2,
  /* o = coef[0] x - coef[1] D; hist[hist_write] = D. DPMPP2SAncestralSampler's midpoint (:279, out = stage) and update
   * (:281, evaluated at xe = stage), DPMPP2MSampler's x_standard (:332, first step and sigma_next = 0). */
  PN_SAMPLER_DPM = 3,
  /* o = coef[0] x - coef[1] (coef[2] D - coef[3] hist[hist_read[0]]); hist[hist_write] = D: DPMPP2MSampler (:337-338). */
  PN_SAMPLER_DPM_2M = 4,
  /* o = coef[0] x, no network term (net unused): prepare_sampling_loop's x *= sqrt(1 + sigma_0^2) (:50), plus the
   * churn noise of step 0 and the first network input. */
  PN_SAMPLER_SCALE = 5
};

typedef struct pn_sampler_step_args {
  float* x;                 /* [n] sampler state */
  const float* x_eval;      /* [n] evaluation point, or NULL = x */
  const float* net;         /* [halves * n] network output (eps; or D when net_is_denoised) */
  float* out;               /* [n] destination of o, or NULL = x (may alias x or x_eval) */
  float* hist;              /* [slots * n] history ring, or NULL */
  const float* noise;       /* [n] caller's standard-normal draws, or NULL = in-kernel Philox */
  float* x_in_next;         /* [halves * n] next network input, or NULL */
  int64_t n;                /* elements of one half */
  uint64_t seed, draw;      /* Philox key and draw index */
  int32_t mode;             /* pn_sampler_mode */
  int32_t halves;           /* 2: VanillaCFG, 1: IdentityGuider */
  int32_t net_is_denoised;
  int32_t hist_read[3];     /* slots read (HEUN, DPM_2M: [0]; LMS: d_{i-1}, d_{i-2}, d_{i-3}); -1 = none */
  int32_t hist_write;       /* slot written (d or D, see the modes); -1 = none */
  float sigma_q;            /* sigma snapped to the denoiser's table: c_out = -sigma_q */
  float cfg_scale;
  float sigma;              /* divisor of to_d */
  float dt;
  float coef[4];            /* LMS coefficients / DPM++ multipliers / SCALE factor */
  float noise_scale, noise_amp;
  float c_in_next;          /* c_in of the next evaluation's quantised sigma */
} pn_sampler_step_args;

int pn_sampler_step(const pn_sampler_step_args* args, void* stream);

/* pn_sampler_step_known — pn_sampler_step with the state blended toward a known latent (editing a recorded clip,
 * DESIGN.md section 13). After the mode's update and the launch's own noise term, per element:
 *   kn = sigma != 0 ? known[e] + sigma * xi : known[e]    xi = the Philox normal of (seed, draw, e), as above; the
 *                                                          product and the sum are each rounded once (no FMA)
 *   o  = m == 1 ? o : m == 0 ? kn : m * o + (1 - m) * kn   m = mask[frame(e) * plane + e % plane]
 * with frame(e) = e / (channels * plane): x is [frames, channels, h, W] and the mask [frames, h, W] (plane = h * W)
 * holds one weight per latent pixel for all its channels. Then out / x and x_in_next are written from the blended o;
 * hist keeps what the mode writes. `sigma` is the noise level of the state the launch leaves in x. */
typedef struct pn_sampler_known_args {
  const float* known;       /* [n] the known latent */
  const float* mask;        /* [n / channels] weights in [0, 1]: 1 keeps the sampler's value, 0 takes the known one */
  int64_t plane;            /* h * W latent pixels of one channel of one frame */
  int32_t channels;         /* latent channels sharing one mask value (n % (channels * plane) == 0) */
  uint64_t seed, draw;      /* Philox key and draw index of the known region's noise */
  float sigma;              /* s above */
} pn_sampler_known_args;

int pn_sampler_step_known(const pn_sampler_step_args* args, const pn_sampler_known_args* known, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Layout maps: the ControlNet's 19-channel hint [frames, 19, H, 6w] (fp32, values k/255) of one clip, rendered from
 * per-panel primitive lists (panacea_b200/layout.py builds them; DESIGN.md section 12). The reference renders the same
 * channels with OpenCV in its dataset (sgm/data/nuscenes_video/nuscenes_datasets_video.py:286-412).
 *  prims          [n, PN_LAYOUT_PRIM_FLOATS] fp32, 16-byte aligned, grouped by panel (frame-major, 6 panels per
 *                 frame). A record is {kind, key, c0, c1, c2, radius, 0, 0, p0.x, p0.y, p1.x, p1.y, p2.x, p2.y, p3.x,
 *                 p3.y}; a RECT is {kind, class, value, -, -, -, 0, 0, x0, y0, x1, y1, ...} (half-open pixel range).
 *  panel_offsets  [frames * 6 + 1] int32: the records of panel i are prims[panel_offsets[i] .. panel_offsets[i+1]).
 *  rays           [6 * 12 + 2] fp64: per panel the first three rows of its img2lidar matrix, then the global min and
 *                 max of the ray components over all panels.
 * Channels 0..2 take the colour of the highest-keyed QUAD or BOX_SEGMENT covering a pixel, 13..15 that of the
 * highest-keyed MAP_SEGMENT, channel 3 + class the minimum value of the RECTs of that class (255 where none).
 * The output is bitwise the same from call to call. */
enum pn_layout_kind { PN_LAYOUT_RECT = 0, PN_LAYOUT_QUAD = 1, PN_LAYOUT_BOX_SEGMENT = 2, PN_LAYOUT_MAP_SEGMENT = 3 };
#define PN_LAYOUT_PRIM_FLOATS 16

int pn_render_layout(const float* prims, const int32_t* panel_offsets, const double* rays, float* out, int64_t frames,
                     int64_t height, int64_t view_width, void* stream);

/* Where two renders of a clip differ, at latent resolution (DESIGN.md section 13). a, b fp32 [frames, 19, H, 6w];
 * out fp32 [frames, H / cell, 6w / cell] in {0, 1}: 1 where any channel of any pixel of the cell differs between a and
 * b, or of a cell of the same panel within Chebyshev distance `dilate` (the dilation stops at panel borders). cell is
 * a power of two <= 32 that divides H and w (8, the VAE factor, for the editing path); (H / cell) * (w / cell) <=
 * 49152. Two launches (compare and pool, then dilate in place); the output is bitwise the same from call to call. */
int pn_layout_change_mask(const float* a, const float* b, float* out, int64_t frames, int64_t height, int64_t view_width,
                          int64_t cell, int64_t dilate, void* stream);

/* A user-drawn edit mask at latent resolution (DESIGN.md section 13). pixels uint8 [frames, H, 6w], nonzero = regenerate;
 * out fp32 [frames, H / cell, 6w / cell] in {0, 1}: 1 where any pixel of the cell is nonzero, dilated by `dilate` cells
 * within each panel exactly as pn_layout_change_mask dilates. Same limits as pn_layout_change_mask. */
int pn_mask_cells(const uint8_t* pixels, float* out, int64_t frames, int64_t height, int64_t view_width, int64_t cell,
                  int64_t dilate, void* stream);

/* Paste the recorded pixels back outside an edit (DESIGN.md section 13). decoded, recorded, out fp32 [frames, 3, H, 6w];
 * cells fp32 [frames, H / cell, 6w / cell], a cell > 0 is regenerated; alpha fp32 [frames, H, 6w] or NULL. For pixel
 * (y, x) of panel v, with R the regenerated cells of the same frame and panel (nothing crosses a panel seam):
 *   d2    = min over c in R of dx^2 + dy^2, dx = max(0, c.x0 - x, x - c.x1) (c.x0, c.x1 its first and last pixel
 *           column; dy likewise with rows): the squared distance between pixel centres, an integer;
 *   alpha = 1 if d2 = 0; 0 if R is empty; else max(0, 1 - sqrt(d2) / (feather + 1)), each operation IEEE fp32;
 *   b     = clamp(rint((recorded + 1) * 127.5), 0, 255), k = (b + 0.5) / 127.5 - 1 (fp32): the recorded byte's centre,
 *           which the writers' truncating quantiser maps back to b;
 *   out   = decoded where alpha = 1, k where alpha = 0 (both bitwise), else k + alpha * (decoded - k), no FMA.
 * cell is a power of two <= 32 that divides H and w, 0 <= feather <= 64; out and alpha alias nothing. One launch; the
 * output is bitwise the same from call to call. */
int pn_composite_frames(const float* decoded, const float* recorded, const float* cells, float* out, float* alpha,
                        int64_t frames, int64_t height, int64_t view_width, int64_t cell, int64_t feather, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PANACEA_B200_H */

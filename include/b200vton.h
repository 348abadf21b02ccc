/* libb200vton.so — C ABI of the Hopper-native (sm_90a) IDM-VTON denoising engine.
 *
 * The reference (yisol/IDM-VTON) has no C/FFI plugin API; its seams are Python protocols (SURVEY.md 8b: pipeline
 * __call__, UNet2DConditionModel.forward, the diffusers attention-processor protocol). This header is the boundary the
 * Python host (idm-vton_b200/*.py, loaded with ctypes) binds instead of the ATen/cuDNN/cuBLAS/SDPA library calls the
 * reference issues. Every entry point cites the reference call site it replaces.
 *
 * Conventions
 *   - all pointers are DEVICE pointers to fp16 data unless stated; the caller (PyTorch) owns every buffer;
 *     the library never allocates or frees device memory;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream); launches are asynchronous and may be
 *     captured into a CUDA graph;
 *   - return value 0 = success, non-zero = error (1 invalid argument, 2 CUDA error, 3 unsupported shape);
 *     b200vton_last_error() returns the message for the calling thread. There is no CPU fallback.
 *   - activations are NHWC / token-major: a feature map [B,H,W,C] and a token matrix [B*H*W, C] are the same memory.
 */
#ifndef B200VTON_H_
#define B200VTON_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int b200vton_version(void);
const char* b200vton_last_error(void);
/* kernels launched (or recorded into a capturing stream) by this library since it was loaded */
long long b200vton_launch_count(void);
/* library options: "programmatic_launch" = 1 launches the hot kernels with programmatic stream serialization (their
 * set-up overlaps the previous kernel's tail; they wait for it before touching global memory); 0 (default) = plain
 * stream order. "gemm_2cta_auto", "gemm_cluster4", "attention_pingpong", "attention_q_tiles" and "attention_poly_exp"
 * select kernel variants of other GPU generations; they are accepted and have no effect (one GEMM and one attention
 * kernel on sm_90a). */
int b200vton_set_option(const char* name, int value);

/* out[M,N] = epi(A[M,K] . W[N,K]^T): nn.Linear on the hot path — attn to_q/to_k/to_v/to_out
 * (ip_adapter/attention_processor.py:240-268), Transformer2DModel.proj_in/proj_out
 * (src/transformerhacked_tryon.py:331-345,410-427), FeedForward GEGLU / net.2 (src/attentionhacked_tryon.py:621-679).
 * epi: v = fp16(acc + bias[n]); v = fp16(v + rowvec[m / rows_per_sample, n]); v = fp16(v + residual[m, n]).
 * flags & 1 (GEGLU): W/bias rows are tile-interleaved [value | gate] (see engine.pack_geglu) and
 *             out[M, N/2] = fp16(value) * fp16(gelu_erf(fp16(gate))).
 * flags & 2 (GELU): v = fp16(gelu_erf(fp16(acc + bias))) before the rowvec / residual terms (ip_adapter/resampler.py:13-20;
 *             the CLIP ViT-H / bigG MLPs). flags & 4 (quick-GELU): v = fp16(x * sigmoid(1.702 x)), x = fp16(acc + bias)
 *             (the CLIP ViT-L text encoder's MLP, src/tryon_pipeline.py:592).
 * K % 64 == 0; N, lda, ldw, ldo % 8 == 0. force_bn: 0 = automatic tile width; 64/128/160/256 = that tile width;
 * 1000 + width and 2000 + width select the same width (encodings of multi-CTA variants). */
int b200vton_gemm_f16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out, int64_t ldo, int M, int N,
                      int K, const void* bias, const void* residual, int64_t ldr, const void* rowvec,
                      int64_t ld_rowvec, int rows_per_sample, int flags, int force_bn, void* stream);

/* FP8 linear (opt-in, UNetEngine(fp8=True)): out[M,N] = epi((acc * a_scale[m]) * w_scale[n]), acc = A_q[M,K] . W_q[N,K]^T
 * over e4m3 (float8_e4m3fn) operands with fp32 accumulation; a_scale [M] fp32 per row (token), w_scale [N] fp32 per
 * output channel (row of W_q). epi is b200vton_gemm_f16's fp16 epilogue on the scaled value: bias, GEGLU (flags & 1, W_q
 * / w_scale / bias rows tile-interleaved as for b200vton_gemm_f16) and residual, at the same fp16 rounding points; no
 * other flag. K % 128 == 0; lda / ldw (elements = bytes) multiples of 16; N, ldo, ldr % 8 == 0; A_q, W_q, out, bias,
 * residual 16-byte aligned, a_scale 4-byte, w_scale 8-byte. force_bn as for b200vton_gemm_f16. */
int b200vton_gemm_e4m3(const void* A_q, int64_t lda, const void* a_scale, const void* W_q, int64_t ldw,
                       const void* w_scale, void* out, int64_t ldo, int M, int N, int K, const void* bias,
                       const void* residual, int64_t ldr, int flags, int force_bn, void* stream);

/* NHWC 3x3 convolution, pad 1, stride 1 or 2, as implicit GEMM: diffusers ResnetBlock2D.conv1/conv2 (+conv_shortcut),
 * conv_in / conv_out (src/unet_hacked_tryon.py:416,755,1245,1386), the conv of Upsample2D, and (stride 2) the conv of
 * Downsample2D (src/unet_block_hacked_tryon.py:1113,1246): the A operand's tensor map then steps two input pixels per
 * output pixel (TMA traversal stride), so no im2col buffer exists.
 * x: [B,H,W,Cin] with channel stride ldx; w: [9][Cout][Cin] (tap = ky*3+kx); out: [B*Ho*Wo, ldo], Ho = (H-1)/stride+1.
 * epi: v = fp16(acc + bias); v = fp16(v + temb[b, n]) (time_emb_proj broadcast add);
 *      1x1 shortcut (w_sc [Cout, C0+C1] over the channel concat of sc0|sc1, accumulated in a second register accumulator):
 *      s = fp16(acc_sc + bias_sc); v = fp16(s + v);   identity residual: v = fp16(v + residual[m, n]). */
int b200vton_conv3x3_nhwc(const void* x, int64_t ldx, int B, int H, int W, int Cin, const void* w, int Cout,
                          const void* bias, const void* temb, int64_t ld_temb, const void* sc0, int C0,
                          const void* sc1, int C1, const void* w_sc, const void* bias_sc, const void* residual,
                          int64_t ldr, void* out, int64_t ldo, int force_bn, int stride, void* stream);

/* softmax(Q K^T * scale) V, head_dim 64, keys/values streamed from two segments without concatenation:
 * segment 0 = (k0, v0)[b]; segment 1 = (k1, v1)[base + (b - kv1_off) % mod] for b >= kv1_off, where mod = kv1_mod
 * (or B1 when kv1_mod == 0) and base = *kv1_base (a device int32, or 0 when NULL: lets one captured graph walk the
 * per-timestep slices of garment K/V precomputed for all denoise steps); for b < kv1_off the N1
 * tokens are all-zero K/V handled in closed form (CFG-uncond half, src/tryon_pipeline.py:1796).
 * Replaces cat + F.scaled_dot_product_attention of src/attentionhacked_tryon.py:334-348 /
 * ip_adapter/attention_processor.py:238-262 (attn1) and :1970-1995 (attn2: call once for the 77 text tokens, once for
 * the 16 IP tokens with accumulate = 1: out = fp16(out + fp16(result))). Also PerceiverAttention
 * (ip_adapter/resampler.py:49-78; segment 0 = image tokens, segment 1 = latents).
 * q: [B,Nq,*] row stride ldq, head h at columns [64h, 64h+64); same for k/v/out. */
int b200vton_attention(const void* q, int64_t ldq, const void* k0, const void* v0, int64_t ldkv0, const void* k1,
                       const void* v1, int64_t ldkv1, void* out, int64_t ldo, int B, int H, int Nq, int N0, int N1,
                       int B1, int kv1_off, int kv1_mod, const void* kv1_base, float scale, int accumulate,
                       void* stream);

/* b200vton_attention with one segment-1 row per sample: sample b >= kv1_off reads row kv1_rows[b - kv1_off] of the
 * [B1, N1, *] K/V (kv1_rows: device int32 [B - kv1_off], read after the previous kernel of the stream completes, so a
 * captured graph can be replayed with a table rewritten before each replay). A negative entry, or one >= B1, selects
 * the all-zero K/V closed form of the samples b < kv1_off: no K/V is read for it. Lets slots at different denoise steps
 * share one pool of hoisted garment K/V (one page of T rows per garment). Needs segment-1 K/V (N1 > 0, B1 > 0, k1, v1)
 * and 0 <= kv1_off < B; otherwise the arguments and results of b200vton_attention. */
int b200vton_attention_rows(const void* q, int64_t ldq, const void* k0, const void* v0, int64_t ldkv0, const void* k1,
                            const void* v1, int64_t ldkv1, void* out, int64_t ldo, int B, int H, int Nq, int N0, int N1,
                            int B1, int kv1_off, const void* kv1_rows, float scale, int accumulate, void* stream);

/* FP8 garment K/V (opt-in, set_garment_kv_precision("fp8"); INTEGRATION.md, "FP8 garment K/V"). The format of the
 * hoisted garment K/V [rows, Ng, 2C] (K in columns [0, C), V in [C, 2C)): per token and per group of 64 columns (group
 * g < H = head g of K, group H + g = head g of V), with amax = max |x| over the group in fp32,
 *   e = 0 when amax == 0, else the smallest integer with amax <= 448 * 2^e, clamped to e >= -24;
 *   q = e4m3_rn_satfinite(x * 2^-e) (exact product, |.| <= 448);   x' = fp16_rn(float(q) * 2^e).
 * q: [rows, Ng, 2C] e4m3; e: int8 [rows, 2H, lde] (group-major, lde >= Ng a multiple of 16, entries >= Ng are 0).
 *
 * b200vton_quantize_kv_e4m3: x fp16 [M, G*64] (row stride ldx, a multiple of 8; 16-byte aligned), M = rows * Ng ->
 * q e4m3 [M, ldq] (ldq a multiple of 8; 8-byte aligned) and e int8 [rows, G, lde] (lde >= Ng; the padding is written 0).
 * Bit-identical to the rule above. */
int b200vton_quantize_kv_e4m3(const void* x, int64_t ldx, int M, int G, int Ng, void* q, int64_t ldq, void* e,
                              int64_t lde, void* stream);

/* b200vton_attention with segment 1 in the FP8 garment K/V format: k1 / v1 are e4m3 [B1, N1, *] views (row stride ldkv1
 * BYTES, a multiple of 16; 16-byte aligned), e1 the int8 exponents [B1, 2H, lde1] of the same rows (lde1 a multiple of
 * 16, >= N1; 16-byte aligned). The kernel dequantizes each tile by the rule (exact: x' = fp16(q) * fp16(2^e) in one
 * rounding), so the result is b200vton_attention's on the dequantized K/V, bit for bit. kv1_rows (device int32
 * [B - kv1_off], or NULL) selects segment-1 rows as in b200vton_attention_rows and replaces kv1_mod / kv1_base; without
 * it, kv1_mod / kv1_base as in b200vton_attention. Needs N1 > 0, B1 > 0 and 0 <= kv1_off < B; head_dim 64. */
int b200vton_attention_kv8(const void* q, int64_t ldq, const void* k0, const void* v0, int64_t ldkv0, const void* k1,
                           const void* v1, int64_t ldkv1, const void* e1, int64_t lde1, void* out, int64_t ldo, int B,
                           int H, int Nq, int N0, int N1, int B1, int kv1_off, int kv1_mod, const void* kv1_base,
                           const void* kv1_rows, float scale, int accumulate, void* stream);

/* Decoupled cross-attention (attn2 of every transformer block) in one launch:
 *   out = fp16( fp16(softmax(Q Kt^T * scale) Vt) + fp16(ip_scale * fp16(softmax(Q Ki^T * scale) Vi)) ),  head_dim 64,
 * Kt/Vt = [B, Nt <= 80, *] the text tokens (attn2.to_k / to_v), Ki/Vi = [B, Ni <= 16, *] the IP-Adapter image tokens
 * (processor to_k_ip / to_v_ip); Ni = 0 (ki = vi = NULL) is the plain text cross-attention of the garment UNet.
 * Replaces IPAttnProcessor2_0.__call__ (ip_adapter/attention_processor.py: two scaled_dot_product_attention calls and
 * hidden_states + self.scale * ip_hidden_states), called as attn2 at src/attentionhacked_tryon.py:368-380, and
 * AttnProcessor2_0 at src/attentionhacked_garmnet.py:371-383. Same result as two b200vton_attention calls
 * (the second with accumulate = 1), one kernel instead of two. Layouts as b200vton_attention. */
int b200vton_cross_attention(const void* q, int64_t ldq, const void* kt, const void* vt, int64_t ldkv_t, int Nt,
                             const void* ki, const void* vi, int64_t ldkv_i, int Ni, void* out, int64_t ldo, int B,
                             int H, int Nq, float scale, float ip_scale, void* stream);

/* fp32 3x3 convolution, stride 1, zero padding 1, on the TF32 tensor cores (TF32 products, fp32 accumulate, fp32 bias,
 * fp32 out — the arithmetic class PyTorch uses for fp32 cuDNN convolutions by default): the VAE's convolutions
 * (diffusers AutoencoderKL ResnetBlock2D.conv1/conv2, Upsample2D.conv; the reference runs the SDXL VAE in fp32,
 * src/tryon_pipeline.py:913-915,1076-1093). x: [B,H,W,Cin] dense NHWC (= channels_last memory), w: [9][Cout][Cin]
 * (tap-major), bias: [Cout] or NULL, residual: [B,H,W,Cout] fp32 NHWC or NULL — out = (acc + bias) + residual, the
 * ResnetBlock2D's `input_tensor + hidden_states` in the epilogue with torch's rounding; out: [B,H,W,Cout].
 * Cin, Cout multiples of 32, Cout >= 64, W divisible by 8. */
int b200vton_conv3x3_nhwc_f32(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                               const void* residual, void* out, void* stream);

/* The same convolution with fp16 operands: x [B,H,W,Cin] fp16 NHWC (the fp16 output of b200vton_groupnorm_nhwc_f32), w
 * [9][Cout][Cin] fp16; fp32 accumulation, fp32 bias / residual / out. An fp16 operand carries the 10-bit mantissa the TF32
 * tensor core rounds an fp32 operand to (and GroupNorm(+SiLU) outputs are far inside fp16's range), so the arithmetic class is
 * that of the TF32 convolution at half the operand traffic and twice the MMA rate. Cin a multiple of 64. */
int b200vton_conv3x3_nhwc_f16in_f32(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                                    const void* residual, void* out, void* stream);

/* Split operands for fp32-accurate products on the TF32 tensor cores (the VAE mid-block attention, diffusers AutoencoderKL
 * mid_block.attentions[0], exact fp32 in the reference: src/tryon_pipeline.py:913-915,1076-1093):
 * hi = tf32(x * scale), lo = tf32(x * scale - hi), both exactly representable in TF32 (10 mantissa bits, round half up).
 * x: B blocks of per_batch contiguous floats with batch stride stride_b (elements); hi / lo: dense [B, per_batch]. */
int b200vton_split_tf32(const void* x, int64_t stride_b, int B, int64_t per_batch, float scale, void* hi, void* lo,
                        void* stream);
/* Row softmax of fp32 scores [rows, N] (max-subtracted, expf, fp32 sum) written directly as the two TF32 parts of the
 * probabilities: p_hi = tf32(p), p_lo = tf32(p - p_hi); the fp32 probabilities themselves are never stored. N % 4 == 0. */
int b200vton_softmax_split_tf32(const void* scores, int64_t rows, int N, void* p_hi, void* p_lo, void* stream);

/* fp32 GroupNorm(32 groups)(+SiLU) over dense NHWC [B,HW,C] fp32 — the VAE's norms (diffusers AutoencoderKL
 * ResnetBlock2D.norm1/norm2 + SiLU, Attention.group_norm, conv_norm_out), deterministic two-stage statistics.
 * gamma/beta: [C] fp32 or NULL. stats_ws: scratch of stats_ws_doubles doubles, at least 64 * max(B, 1184) is always
 * enough. out: fp32, or — out_fp16 != 0 — fp16 of the same shape (one rounding of the fp32 result), the operand format of
 * b200vton_conv3x3_nhwc_f16in_f32; out must not alias x (no in-place call). The VAE's default route (B200VTON_VAE_NHWC=0 restores the cuDNN NCHW path). */
int b200vton_groupnorm_nhwc_f32(const void* x, int B, int HW, int C, const void* gamma, const void* beta, float eps,
                                 int silu, void* stats_ws, int64_t stats_ws_doubles, void* out, int out_fp16, void* stream);

/* GroupNorm(32 groups) over NHWC [B,HW,C0+C1] read from up to two channel-concatenated sources (x1 may be NULL),
 * fp32 statistics (deterministic fixed-order reduction, no atomics on data), optional SiLU, fp16 out [B*HW, C0+C1].
 * ONE launch: statistics, a per-sample barrier between the CTAs of the launch, and the normalisation (the rows stay in
 * shared memory in between when they fit, so the tensor is read once). B <= 4096.
 * stats_ws: (max(B,296)*64 + 4096) doubles; the last 4096 doubles hold the barrier state and must be ZERO before the
 * first call that uses this workspace (the kernel leaves them reusable: no clearing between calls / graph replays).
 * One workspace must not be shared by launches that may run concurrently (different streams); more generally two
 * GroupNorm launches must not run CONCURRENTLY on one device (two streams, two processes): each sizes its grid to be
 * fully co-resident on an otherwise free device, and two half-resident grids would wait for each other at their
 * barriers (the spin is bounded: the kernel traps after 4 s instead of hanging). The engine launches everything on one
 * stream, like the reference pipeline.
 * diffusers ResnetBlock2D.norm1/norm2 (+nonlinearity), Transformer2DModel.norm
 * (src/transformerhacked_tryon.py:329), conv_norm_out + conv_act (src/unet_hacked_tryon.py:1384-1385). */
int b200vton_groupnorm(const void* x0, int C0, const void* x1, int C1, int B, int HW, const void* gamma,
                       const void* beta, float eps, int silu, void* stats_ws, void* out, void* stream);

/* LayerNorm over the last dim of [rows, C]: BasicTransformerBlock.norm1/2/3
 * (src/attentionhacked_tryon.py:310,365,390); the garment UNet's norm1 output is the exported garment feature
 * (src/attentionhacked_garmnet.py:321-322). */
int b200vton_layernorm(const void* x, int64_t ldx, int rows, int C, const void* gamma, const void* beta, float eps,
                       void* out, int64_t ldo, void* stream);

/* b200vton_layernorm followed by the FP8 linears' row quantization: with y16 the fp16 LayerNorm row (written to out
 * [rows, ldo] when out is not NULL, bit-identical to b200vton_layernorm), amax = max|y16|, q_scale[r] = amax / 448 and
 * q[r, :] = e4m3_rn_satfinite(y16 * (448 / amax)) (fp32 IEEE division and product); an all-zero row stores q_scale 1 and
 * q 0. q: [rows, ldq] e4m3, ldq % 16 == 0; q_scale: [rows] fp32. */
int b200vton_layernorm_e4m3(const void* x, int64_t ldx, int rows, int C, const void* gamma, const void* beta,
                            float eps, void* out, int64_t ldo, void* q, int64_t ldq, void* q_scale, void* stream);

/* dst[s,y,x,c_off+c] = src[s % Bs, c, y, x]: NCHW module inputs -> NHWC engine buffer; implements the CFG
 * duplication and the 13-channel concat of src/tryon_pipeline.py:1769,1777 as batch/channel offsets. */
int b200vton_nchw_to_nhwc(const void* src, int Bs, int Cs, int H, int W, void* dst, int Bd, int ldc, int c_off,
                          void* stream);
/* b200vton_nchw_to_nhwc with dst = fp16(src * scale[0]); scale: one fp32 on device (4-byte aligned, not null). With the
 * reciprocal 1/sqrt(sigma^2 + 1) it is EulerDiscreteScheduler.scale_model_input on the latent channels
 * (src/tryon_pipeline.py:1772, before the channel concat of :1777). */
int b200vton_nchw_to_nhwc_scaled(const void* src, int Bs, int Cs, int H, int W, void* dst, int Bd, int ldc, int c_off,
                                 const void* scale, void* stream);
/* b200vton_nchw_to_nhwc_scaled with one scale per source sample: dst[s, ..] = fp16(src[s % Bs, ..] * scale[s % Bs]);
 * scale: Bs fp32 on device. Rows b and b + Bs of the CFG duplication both use scale[b]: Euler's scale_model_input when
 * every sample is at its own step (continuous batching). Pointers not null; src / dst 2-byte, scale 4-byte aligned. */
int b200vton_nchw_to_nhwc_scaled_rows(const void* src, int Bs, int Cs, int H, int W, void* dst, int Bd, int ldc,
                                      int c_off, const void* scale, void* stream);
/* dst NCHW [B,C,H,W] = src NHWC [B,H,W,ldc][..., :C] */
int b200vton_nhwc_to_nchw(const void* src, int B, int C, int H, int W, int ldc, void* dst, void* stream);

/* nearest-neighbour x2 (diffusers Upsample2D's F.interpolate), NHWC; = b200vton_upsample_nearest_nhwc to (2H, 2W) */
int b200vton_upsample2x_nhwc(const void* src, int B, int H, int W, int C, void* dst, void* stream);
/* nearest-neighbour resize src [B,H,W,C] -> dst [B,Hout,Wout,C], NHWC, C % 8 == 0, src / dst 16-byte aligned: diffusers
 * Upsample2D's F.interpolate(size=upsample_size, mode="nearest") when the UNet forwards an upsample size (latent size not a
 * multiple of 2^num_upsamplers: src/unet_hacked_tryon.py:1081-1091,1357-1379, src/unet_hacked_garmnet.py:994-1000,
 * 1264-1274). Source index per axis as ATen's `nearest` mode: identity when out == in, dst >> 1 when out == 2 in,
 * otherwise min((int)floorf(dst * ((float)in / out)), in - 1). */
int b200vton_upsample_nearest_nhwc(const void* src, int B, int H, int W, int C, int Hout, int Wout, void* dst,
                                   void* stream);
/* patches of a 3x3 stride-2 pad-1 conv (diffusers Downsample2D) as A[B*Ho*Wo, 9*C], K ordered tap-major */
int b200vton_im2col3x3_s2_nhwc(const void* src, int B, int H, int W, int C, void* dst, void* stream);

/* diffusers Timesteps(dim, flip_sin_to_cos=True, freq_shift=0): out[r, :] = [cos | sin](values[r % n] * freq),
 * values: n fp32 on device; out: [n * rows_repeat, dim] fp16 (src/unet_hacked_tryon.py:1134-1139,1185). */
int b200vton_timestep_embedding(const void* values, int n, int dim, int rows_repeat, void* out, void* stream);

/* y = W x + b for M <= 16 rows (TimestepEmbedding, add_embedding, batched ResnetBlock2D.time_emb_proj):
 * x' = in_silu ? fp16(silu(x)) : x; y = fp16(W x' + b); y = out_silu ? fp16(silu(y)) : y; y = fp16(y + addend). */
int b200vton_skinny_linear(const void* x, int ldx, int M, int K, const void* W, int64_t ldw, int N, const void* bias,
                           int in_silu, int out_silu, const void* addend, int ld_add, void* out, int ldo,
                           void* stream);

/* Encoder self-attention for the CLIP towers around the loop (SURVEY.md 8f row 2): replaces transformers' CLIPAttention
 * inside `self.image_encoder(image, output_hidden_states=True)` (src/tryon_pipeline.py:468-470: ViT-H, 16 heads of 80,
 * 257 tokens, no mask) and inside `text_encoder(text_input_ids, output_hidden_states=True)` (src/tryon_pipeline.py:592-596:
 * heads of 64, 77 tokens, causal mask). q / k / v: [B, N, >= H*D] views with row strides ldq / ldkv (the three column
 * blocks of a fused QKV projection buffer); out: [B, N, H*D], row stride ldo. D = 16..96, multiple of 16.
 * out = softmax(scale * q k^T [+ causal mask]) v per head, fp32 softmax, fp16 probabilities, fp32 accumulation. */
int b200vton_encoder_attention(const void* q, int64_t ldq, const void* k, const void* v, int64_t ldkv, void* out,
                               int64_t ldo, int B, int H, int N, int D, float scale, int causal, void* stream);

/* CLIPVisionEmbeddings.patch_embedding as a GEMM operand (src/tryon_pipeline.py:468): x [B,C,Hi,Wi] fp16 ->
 * out [B*(Hi/P)*(Wi/P), ldk] fp16, row = (b, gy, gx), column = (c, ky, kx) = the flattened conv weight's K order;
 * columns >= C*P*P are written as zeros (ldk = K rounded up to a multiple of 64 for b200vton_gemm_f16). */
int b200vton_patchify(const void* x, int B, int C, int Hi, int Wi, int P, void* out, int ldk, void* stream);

/* CLIPTextEmbeddings (src/tryon_pipeline.py:592): out[r, :] = fp16(token_embedding[ids[r], :] + position_embedding[r % T, :]);
 * ids: int64 [rows] on the device (clamped to [0, vocab)); C % 8 == 0. */
int b200vton_token_embedding(const void* ids, int rows, int T, int C, int vocab, const void* token_embedding,
                             const void* position_embedding, void* out, void* stream);

/* CFG combine + DDPMScheduler.step (src/tryon_pipeline.py:1814-1823). eps NHWC [2B,HW,ldc] (uncond first) or [B,..]
 * when do_cfg == 0; latents/noise/out NCHW [B,C,H,W] (noise may be NULL); coef: 6 fp32 on device
 * {guidance_scale, sqrt(1-abar_t), 1/sqrt(abar_t), x0 coeff, x_t coeff, sigma_t}. */
int b200vton_cfg_ddpm_step(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                           const void* noise, const void* coef, int do_cfg, void* out, void* stream);

/* b200vton_cfg_ddpm_step with guidance rescale between the CFG combine and the DDPM step (rescale_noise_cfg,
 * src/tryon_pipeline.py:101-113,1818-1820): per sample, g' = phi * g * std(cond)/std(g) + (1 - phi) * g with unbiased
 * std over C*H*W, in the reference's fp16 rounding points. Same layout as b200vton_cfg_ddpm_step; coef: 7 fp32 on
 * device {the 6 above, phi}. One CTA per sample, deterministic reductions, graph-capturable. do_cfg == 0 runs
 * b200vton_cfg_ddpm_step (no rescale without CFG, as in the reference). */
int b200vton_cfg_rescale_ddpm_step(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                                   const void* noise, const void* coef, int do_cfg, void* out, void* stream);

/* CFG combine + one step of DDIMScheduler (kind 0), EulerDiscreteScheduler with s_churn = 0 (kind 1) or
 * DPMSolverMultistepScheduler, dpmsolver++ / midpoint, order 1 or 2 (kind 2); epsilon prediction. Layout of
 * b200vton_cfg_ddpm_step; coef: 8 fp32 on device {gs, s, inv_a, p, q, r, sigma_n, k}:
 *   x0 = (x - s g) * inv_a;  D = (1 + k/2) x0 - (k/2) x0_prev;  out = p x + q D + r g + sigma_n noise
 * with each scheduler's own rounding points (listed at cfg_solver_kernel in elementwise.cu). x0_prev: [B,C,H,W] fp16,
 * required by kind 2 (read, then overwritten with this step's x0), ignored otherwise. Pointers 2-byte aligned (coef 4). */
int b200vton_cfg_solver_step(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                             const void* noise, void* x0_prev, const void* coef, int kind, int do_cfg, void* out,
                             void* stream);

/* b200vton_cfg_ddpm_step / b200vton_cfg_solver_step with one coefficient row per sample: coef is [B, coef_stride] fp32 on
 * device and sample b reads row b, so every sample of the batch can be at its own denoise step (continuous batching).
 * coef_stride 0 gives every sample row 0, which is the single-row entry point's result bit for bit; otherwise it must be
 * at least the kind's coefficient count (6 for DDPM, 8 for the solver kinds). Same layouts and rounding points as the
 * single-row entry points; eps, latents, coef and out not null; fp16 pointers 2-byte aligned, coef 4-byte. */
int b200vton_cfg_ddpm_step_rows(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                                const void* noise, const void* coef, int coef_stride, int do_cfg, void* out,
                                void* stream);
int b200vton_cfg_solver_step_rows(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                                  const void* noise, void* x0_prev, const void* coef, int coef_stride, int kind,
                                  int do_cfg, void* out, void* stream);

/* One step of a batch whose samples follow different schedulers (sampling presets of continuous batching). Same layout
 * as b200vton_cfg_solver_step_rows, plus kinds: a device int32 array of B entries, read after the kernel's
 * griddepcontrol.wait. Sample b takes kind kinds[b] with coefficient row b:
 *   0 DDIM, 1 Euler, 2 DPM-Solver++ (row {gs, s, inv_a, p, q, r, sigma_n, k}): b200vton_cfg_solver_step_rows' result;
 *   3 DDPM (row {gs, sb, inv_sa, c0, c1, sigma, phi, 0}): b200vton_cfg_ddpm_step_rows' result, or under CFG with
 *     phi > 0 b200vton_cfg_rescale_ddpm_step's result on that sample alone.
 * noise (may be null) enters DDPM and DDIM rows only; x0_prev (required) is read and rewritten by DPM-Solver++ rows only.
 * Kind values are not checked on the device. coef_stride 0 or >= 8; fp16 pointers 2-byte aligned, coef and kinds 4. */
int b200vton_cfg_step_mixed_rows(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                                 const void* noise, void* x0_prev, const void* coef, int coef_stride, const void* kinds,
                                 int do_cfg, void* out, void* stream);

/* Pre-processing of the inpainting inputs in one launch (diffusers VaeImageProcessor.preprocess for image and mask,
 * the masked image and the latent-resolution mask: src/tryon_pipeline.py:1588-1602, 940-943). image: [B,3,H,W] fp32;
 * mask: [B,mask_channels,H,W] fp32 (1, or 3 = RGB converted to grayscale); image_min: device scalar = min(image)
 * (values already in [-1,1], i.e. min < 0, are not normalised again — diffusers' rule, decided on the device);
 * outputs: init_image, masked_image [B,3,H,W] fp32, mask_bin [B,1,H,W] fp32 (0/1 at threshold 0.5),
 * mask_latent [B,1,H/vae_scale,W/vae_scale] fp16 (nearest). */
int b200vton_preprocess_inpaint(const void* image, const void* mask, int mask_channels, const void* image_min, int B,
                                int H, int W, int vae_scale, void* init_image, void* mask_bin, void* masked_image,
                                void* mask_latent, void* stream);

/* Post-processing of the VAE decoder output in one launch (VaeImageProcessor.postprocess, src/tryon_pipeline.py:1885):
 * x [B,3,H,W] fp32 in NCHW memory (nhwc = 0) or NHWC memory (nhwc = 1) -> clamp(x/2 + 0.5, 0, 1) written as fp32 NCHW
 * (out_pt, may be NULL) and/or uint8 NHWC round(255 y) (out_u8, may be NULL; what "np"/"pil" produce, 4x less D2H). */
int b200vton_postprocess_image(const void* x, int nhwc, int B, int H, int W, void* out_pt, void* out_u8, void* stream);

/* Full-resolution photos (INTEGRATION.md, "Full-resolution photos"; the reference demo's auto-crop, resize and
 * paste-back, gradio_demo/app.py:135-147, 236-239). Both entry points are integer-only and deterministic.
 *
 * b200vton_resample_u8: Pillow's Image.resize with a convolution filter (ImagingResample, 8 bits per channel) of a
 * batch of uint8 HWC crops (channels 1 or 3), each with its own sizes. The crop [crop_x, crop_x + crop_w) x
 * [crop_y, crop_y + crop_h) of `src` is the image: taps are clipped to the crop, never to the photo around it.
 * Per axis, `tables` holds at bounds_* two int32 per output (first tap, tap count) and at coefs_* ksize_* int32 per
 * output: Pillow's coefficients (precompute_coeffs) in 22-bit fixed point (normalize_coeffs_8bpc). need_x / need_y
 * say whether Pillow runs that pass (output size != crop size on that axis). The horizontal pass runs first:
 *   tmp[r][x] = clip8(2^21 + sum_k src[tmp_first + r][first_x + k] * coef_x[k]),   r < tmp_rows,
 * into `workspace` at tmp_offset (tmp_rows x out_w x channels bytes; tmp_first..tmp_first + tmp_rows are the crop rows
 * the vertical pass reads), then the vertical pass on tmp (or on the crop when need_x == 0):
 *   dst[y][x] = clip8(2^21 + sum_k tmp[first_y - tmp_first + k][x] * coef_y[k]),   clip8(s) = clamp(s >> 22, 0, 255).
 * With neither pass the crop is copied. out_f32 (may be NULL) receives the result as fp32 NCHW [channels, out_h, out_w]:
 * f32_mode 0 = v / 255 (np.asarray(img, np.float32) / 255), 1 = (v / 255 - 0.5) / 0.5 (ToTensor + Normalize(0.5, 0.5)).
 * descs (host) is checked and sizes the grid; descs_dev is the same table in device memory, read by the kernels. The
 * table contents (first taps and counts within the crop, as Pillow's bounds are) are not checked. Two launches (one per
 * pass), each covering the whole batch. n <= 4096. */
typedef struct b200vton_resample_desc {
  const uint8_t* src;
  int64_t src_pitch;  /* bytes per row */
  int32_t src_w, src_h, crop_x, crop_y, crop_w, crop_h;
  uint8_t* dst;
  int64_t dst_pitch;
  float* out_f32;
  int32_t out_w, out_h, channels, f32_mode;
  int32_t bounds_x, coefs_x, ksize_x, need_x;
  int32_t bounds_y, coefs_y, ksize_y, need_y;
  int64_t tmp_offset;
  int32_t tmp_first, tmp_rows;
} b200vton_resample_desc;
int b200vton_resample_u8(const b200vton_resample_desc* descs, const void* descs_dev, int n, const int32_t* tables,
                         int64_t table_len, void* workspace, int64_t workspace_bytes, void* stream);

/* b200vton_paste_u8: the full-resolution results of a batch of photos (uint8 HWC, 3 channels) in one launch:
 * dst = photo outside the box [box_x, box_x + box_w) x [box_y, box_y + box_h); inside it image[y - box_y][x - box_x]
 * (the resampled output, box_w x box_h x 3), or, with a mask (1 channel, mask_w x mask_h at (mask_x, mask_y) in photo
 * coordinates, covering the box), image where mask >= 128 and photo elsewhere. dst may not alias photo or image. */
typedef struct b200vton_paste_desc {
  const uint8_t* photo;
  int64_t photo_pitch;
  uint8_t* dst;
  int64_t dst_pitch;
  const uint8_t* image;
  int64_t image_pitch;
  const uint8_t* mask;
  int64_t mask_pitch;
  int32_t width, height, box_x, box_y, box_w, box_h;
  int32_t mask_x, mask_y, mask_w, mask_h;
} b200vton_paste_desc;
int b200vton_paste_u8(const b200vton_paste_desc* descs, const void* descs_dev, int n, void* stream);

/* b200vton_clip_pixels_u8: CLIPImageProcessor's centre crop, rescale and normalize (INTEGRATION.md, "Garment photos and
 * descriptions") of a batch of uint8 HWC RGB images already resampled to the CLIP size (short side 224), in one launch:
 *   out[j][c][y][x] = table[c * 256 + src_j[crop_y + y][crop_x + x][c]],   0 <= x, y < 224,
 * out fp32 NCHW [n, 3, 224, 224]. table: 3 x 256 fp32 in device memory (per channel, float32((float64(v) / 255 - mean)
 * / std) as transformers computes it). Each descriptor has its own size and crop origin; the 224 x 224 crop must lie
 * inside the image. descs (host) is checked; descs_dev is the same table in device memory, read by the kernel.
 * n <= 4096. */
#define B200VTON_CLIP_SIZE 224
typedef struct b200vton_clip_desc {
  const uint8_t* src;
  int64_t src_pitch;  /* bytes per row */
  int32_t src_w, src_h, crop_x, crop_y;
} b200vton_clip_desc;
int b200vton_clip_pixels_u8(const b200vton_clip_desc* descs, const void* descs_dev, int n, const float* table,
                            float* out, void* stream);

/* b200vton_freeu_nhwc: FreeU (diffusers `apply_freeu`, https://arxiv.org/abs/2309.11497) before one resnet of the
 * try-on UNet's up stage 0 or 1 (src/unet_block_hacked_tryon.py:2322-2344,2458-2480), in one launch:
 *   hidden[..., c] = fp16(float(hidden[..., c]) * b) for c < Ch / 2, in place (channels Ch / 2.. keep their bits);
 *   skip_out = fourier_filter(skip, threshold=1, scale=s): the 2-D spectrum of every (sample, channel) plane times s at
 *   the frequencies {0, -1} along each axis ({0} along an axis of size 1), computed in closed form in fp32 from the
 *   fp16 input (7 sums per channel in a fixed order, then one pass) and rounded to fp16 once.
 * hidden [B,H,W,Ch], skip / skip_out [B,H,W,Cs], NHWC fp16, contiguous, 16-byte aligned; Ch % 8 == 0, Cs % 8 == 0.
 * skip_out may be skip (in place) or must not overlap it; hidden may overlap neither. */
int b200vton_freeu_nhwc(void* hidden, int Ch, const void* skip, void* skip_out, int Cs, int B, int H, int W, float b,
                        float s, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200VTON_H_ */

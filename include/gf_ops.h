/*
 * gf_ops.h -- C ABI of the memory-bound companions of the attention hot path (SURVEY.md row f3).
 *
 * sm_90a equivalents of the reference's two native CUDA ops -- dnnlib/tflib/ops/fused_bias_act.cu and
 * dnnlib/tflib/ops/upfirdn_2d.cu (expected upstream locations; NOT in the reference checkout,
 * /root/reference/.SUBMODULES.json:2) -- restricted to the uses the generator makes of them, plus the
 * activation-scaling form of StyleGAN2's weight (de)modulation.  Channels-last fp32, raw device pointers,
 * enqueue-only on `stream` (a cudaStream_t passed as void*), same error convention as gf_attn.h.
 *
 * Alignment: the channels-last kernels move float4s.  Every operand listed as "16-byte aligned" below must start on a 16-byte
 * boundary (a contiguous view that starts 4 bytes into its storage does not); otherwise the call returns GF_ERR_INVALID
 * before it touches the device.
 */
#ifndef GF_OPS_H_
#define GF_OPS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* y[b,t,c] = x[b,t,c] * s[b*s_ld + c].   Style modulation of a conv input / demodulation of a conv output
 * (modulated_conv2d_layer in the reference, activation-scaling form).  y may alias x.  C % 4 == 0; s_ld (row stride
 * of s in floats) % 4 == 0 so that rows of a column slice of a wider [B, sum C] style matrix can be passed directly.
 * x, s and y 16-byte aligned. */
int gf_chan_scale_nhwc(const float* x, const float* s, int s_ld, float* y, int B, int HW, int C, void* stream);

/* upfirdn_2d, use (a): the FIR blur that follows a stride-2 transposed convolution.
 * x [B, Hout+1, Wout+1, C] -> y [B, Hout, Wout, C]; separable filter [1,3,3,1]/8 per axis, total gain `gain`
 * (4 after an upsampling conv), zero padding 1 on every side; optional per-(b,c) scale (demodulation). C % 4 == 0.
 * x, y and scale 16-byte aligned. */
int gf_blur_up_nhwc(const float* x, float* y, const float* scale, int B, int Hout, int Wout, int C, float gain, void* stream);

/* Use (a) again, with the transposed convolution's output T [B, Hout+1, Wout+1, C] given as its four polyphase components
 * pab[b, i, j, c] = T[b, 2i+a, 2j+b', c] (p00 [B,H+1,W+1,C], p01 [B,H+1,W,C], p10 [B,H,W+1,C], p11 [B,H,W,C]; H = Hout/2,
 * W = Wout/2): the stride-2 transposed 3x3 convolution equals four stride-1 convolutions of the low-resolution input
 * (2x2, 2x1, 1x2 and 1x1 taps), which cuDNN runs 1.3-1.7x faster than its strided dgrad; they are never interleaved.
 * The four phases, y and scale 16-byte aligned. */
int gf_blur_up_phases_nhwc(const float* p00, const float* p01, const float* p10, const float* p11, float* y, const float* scale,
                           int B, int Hout, int Wout, int C, float gain, void* stream);

/* upfirdn_2d, general stride-1 form with the [1,3,3,1]^2/64 filter and symmetric zero padding `pad` in 0..3:
 * x [B,Hin,Win,C] -> y [B,Hin+2*pad-3,Win+2*pad-3,C] times `gain`.  pad 1 = use (a); pad 2 = its adjoint (the backward pass:
 * the filter is symmetric, so d/dx of a pad-p blur is a pad-(3-p) blur of the incoming gradient) and the blur in front of the
 * discriminator's stride-2 3x3 convolutions; pad 1 also serves the discriminator's 1x1 skip path.  C % 4 == 0.
 * x and y 16-byte aligned. */
int gf_fir4_nhwc(const float* x, float* y, int B, int Hin, int Win, int C, int pad, float gain, void* stream);

/* upfirdn_2d, use (b): 2x upsampling of an NCHW image (skip connection of the tRGB outputs):
 * zero-insert, pad (2,1,2,1), FIR [1,3,3,1]^2/64 * 4.  y [B,C,2H,2W] = up(x [B,C,H,W]) (+ add, nullable, same shape as y). */
int gf_upsample2x_nchw(const float* x, const float* add, float* y, int B, int C, int H, int W, void* stream);

/* fused_bias_act (+ the noise input of the synthesis layer):
 *   y = act(x + noise[b*noise_bstride + t] * (*strength) + bias[c]) * gain
 * act: 0 linear, 1 leaky-ReLU(0.2).  noise / strength / bias nullable.  y may alias x.  C % 4 == 0.
 * x, y and bias 16-byte aligned. */
int gf_bias_act_nhwc(const float* x, float* y, const float* bias, const float* noise, const float* strength,
                     long long noise_bstride, int B, int HW, int C, int act, float gain, void* stream);

/* StyleGAN2 demodulation coefficients of the activation-scaling form:
 *   d[b,o] = rsqrt( sum_i styles[b*s_ld + i]^2 * wsq[o,i] + eps ),  wsq[o,i] = sum_{kh,kw} w_eff[o,i,kh,kw]^2 */
int gf_demod_coef(const float* styles, int s_ld, const float* wsq, float* d, int B, int O, int I, float eps, void* stream);

/* The same for every convolution layer of a network in ONE launch (the layers' style vectors all come from one latent, so their
 * demodulation coefficients can be computed up front): n <= GF_DEMOD_MAX_JOBS jobs, common batch B. */
#define GF_DEMOD_MAX_JOBS 32
typedef struct gf_demod_job {
  const float* styles;   /* [B][s_ld], I used */
  const float* wsq;      /* [O][I] */
  float* d;              /* [B][O] out */
  int32_t s_ld, O, I, pad_;
} gf_demod_job;
int gf_demod_coef_batch(const gf_demod_job* jobs, int n, int B, float eps, void* stream);

/* tRGB (SURVEY row f4): 1x1 modulated convolution WITHOUT demodulation from channels-last activations to a planar image,
 *   y[b,o,t] = sum_c x[b,t,c] * w[o*C + c] * styles[b*s_ld + c] * wscale + bias[o],   o < 3
 * (modulated_conv2d_layer(..., demodulate=False, kernel=1) + bias of the reference's torgb); x is read once.
 * C % 4 == 0, C <= 512; s_ld % 4 == 0; bias nullable; x, w and styles 16-byte aligned. */
int gf_torgb_nhwc(const float* x, const float* w, const float* styles, int s_ld, const float* bias, float wscale, float* y,
                  int B, int HW, int C, void* stream);

/* gf_torgb_nhwc with a second output from the same read of x: xs_out[b,t,c] = x[b,t,c] * s2[b*s2_ld + c] -- the style modulation
 * of the NEXT block's first convolution (replaces a gf_chan_scale_nhwc pass over the same tensor).  s2 / xs_out both NULL or both
 * given, both 16-byte aligned. */
int gf_torgb_scale_nhwc(const float* x, const float* w, const float* styles, int s_ld, const float* bias, float wscale, float* y,
                        const float* s2, int s2_ld, float* xs_out, int B, int HW, int C, void* stream);

/* G_mapping (SURVEY row f4) as one kernel: z [B, k+1, D] -> out [B, k+1, D].  Every latent is pixel-normalised
 * (x * rsqrt(mean x^2 + 1e-8)), then runs through L fully connected layers with leaky-ReLU(0.2) -- path 0 (shared by the k local
 * components) or path 1 (the last, global latent) -- and, when w_avg [2, D] is given, the truncation lerp
 * out = w_avg[path] + psi * (y - w_avg[path]).  w [2, L, D(in), D(out)] and b [2, L, D] are the EFFECTIVE weights (equalised-LR
 * scale lr_mul/sqrt(D), bias scale lr_mul and the activation gain sqrt(2) folded in: lrelu(g x) = g lrelu(x)).
 * Replaces the reference's G_mapping dense_layer chain.  D <= 128 and 2*L*D*D floats must fit shared memory. */
int gf_mapping_fwd(const float* z, const float* w, const float* b, const float* w_avg, float psi, float* out,
                   int B, int k, int D, int L, void* stream);

/* Class-conditional G_mapping (SURVEY A.4 item 14) as one kernel: gf_mapping_fwd with labels c [B, c_dim] and the label
 * embedding E [c_dim, D].  Image b's embedding e_b = c_b E is concatenated to each of its k+1 latents, and every row
 * [z_bj || e_b] is pixel-normalised over its 2D entries.  Layer 0 of both paths takes that 2D input: w0 [2, 2D(in), D(out)]
 * (gain lr_mul/sqrt(2D), times sqrt(2), folded in).  Layers 1..L-1 are w [2, L-1, D, D] as in gf_mapping_fwd (NULL when L == 1);
 * b [2, L, D] holds the biases of all L layers.  Zero label entries are skipped, so a one-hot label reads one row of E.
 * E and the label half of w0 are read through L2; the rest of the weights are staged in shared memory, the same 2*L*D*D floats
 * as gf_mapping_fwd, so the two serve the same shapes.  c_dim >= 1, D <= 128. */
int gf_mapping_fwd_cond(const float* z, const float* c, int c_dim, const float* E, const float* w0, const float* w, const float* b,
                        const float* w_avg, float psi, float* out, int B, int k, int D, int L, void* stream);

/* Row f1, first kernel: the 3x3 stride-1 convolution of the synthesis layers (zero padding 1) as a wgmma implicit GEMM in TF32,
 * channels-last: y[b,h,w,o] = sum_{dy,dx,i} x[b,h+dy-1,w+dx-1,i] * wt[dy*3+dx][o][i].  This is the convolution inside the reference's
 * modulated_conv2d_layer in its activation-scaling form (x already carries the style, demodulation is applied by the consumer).
 * wt comes from gf_conv3x3_pack_weights (w [Cout,Cin,3,3] * scale -> [9][Cout][Cin], rounded to TF32).
 * B, H, W > 0, H % 8 == 0, W % 16 == 0, Cin % 32 == 0, Cout % 64 == 0; 16-byte aligned pointers. */
int gf_conv3x3_pack_weights(const float* w, float* wt, int Cout, int Cin, float scale, void* stream);
int gf_conv3x3_nhwc_tf32(const float* x, const float* wt, float* y, int B, int H, int W, int Cin, int Cout, void* stream);

/* Row f1, the upsampling layers: stride-2 transposed 3x3 convolution + FIR blur (use (a) above) + demodulation in one wgmma kernel,
 * TF32, channels-last.  x [B,H,W,Cin] -> y [B,2H,2W,Cout] =
 *   gain * scale[b,o] * blur(conv_transpose2d(x, w^T, stride 2))
 * with wt = gf_conv3x3_pack_weights of the UN-transposed w [Cout,Cin,3,3].  H, W are the input size (any positive value);
 * Cin % 32 == 0, Cout % 64 == 0; 16-byte aligned pointers. */
int gf_upconv3x3_blur_nhwc_tf32(const float* x, const float* wt, const float* scale, float* y, int B, int H, int W, int Cin, int Cout,
                                float gain, void* stream);

/* Adaptive discriminator augmentation (SURVEY A.4 item 15): ADA's integer "pixel blitting" and a per-image colour matrix in one
 * pass over an NCHW fp32 image (csrc/gf_augment.cu).  x, y [B, C, H, W]:
 *   y[b,c,y,x] = sum_j M_b[c][j] x[b,j,R_H(sy),R_W(sx)] + M_b[c][3]   (colour given; without it y[b,c,..] = x[b,c,R_H(sy),R_W(sx)])
 * with (sx, sy) = D_b(x, y) - (tx_b, ty_b) and R_N the mirror that does not repeat the edge pixel: R_N(i) = -i for i < 0,
 * 2(N-1) - i for i >= N.
 *   geom  int32 [B, 4] = (code, tx, ty, unused).  D_b = rotation by k*90 degrees (k = code >> 1) after an x flip (code bit 0):
 *         code 0..7 are the 8 dihedral maps of the grid onto itself.
 *   color float [B, 12] = M_b, a row-major 3x4 matrix applied to (r, g, b, 1); NULL: geometry only.
 * The parameters live on the device, so the kernels define every stored value: the code is masked to 3 bits, and when H != W its
 * bit 1 is cleared (rotations by 90 / 270 degrees would transpose the grid, so they fall back to 0 / 180); tx and ty are clamped to
 * [-(W-1), W-1] and [-(H-1), H-1], so one reflection brings every index back onto the grid.
 * Errors, before touching the device: GF_ERR_INVALID for a NULL x / y / geom or a size <= 0; GF_ERR_UNSUPPORTED for H or W < 2,
 * a colour matrix with C != 3, and H or W > 32768 or C*H*W >= 2^31.  y must not alias x. */
int gf_augment_nchw(const float* x, float* y, const int* geom, const float* color, int B, int C, int H, int W, void* stream);

/* The adjoint of gf_augment_nchw's linear part: gx = A^T gy, the transposed 3x3 colour matrix (the offset column does not take
 * part) followed by the adjoint of the blit.  The mirror lets one source pixel be read by up to 2 outputs per axis; every source
 * pixel gathers its preimages and sums them in a fixed order, without atomics, so the result is the same bits on every run and
 * under CUDA-graph replay.  Same arguments, parameter rules and errors as gf_augment_nchw; gx must not alias gy. */
int gf_augment_adjoint_nchw(const float* gy, float* gx, const int* geom, const float* color, int B, int C, int H, int W, void* stream);

/* ADA's general geometry (SURVEY A.4 item 16): gf_augment_nchw with, per image, a fractional inverse map
 *   frac  float [B, 6] = F_b^-1, a row-major 2x3 affine map in centred pixel coordinates (pixel (i, j) sits at (j - (W-1)/2, i - (H-1)/2)).
 * An image whose F_b^-1 is exactly the identity is blitted, bit for bit as gf_augment_nchw.  Every other image reads the source at
 * B_b^-1(F_b^-1(u)), B_b^-1(v) = D_b v - t_b the blit of geom[b], through ADA's band-limited resampler: mirror extension by R_N to
 * [-(N-1), 2(N-1)] per axis (zeros beyond), 2x upsampling with the 12-tap sym6 low-pass (normalised to sum 1, a convolution, gain 2
 * per axis, pads (6, 5)), bilinear sampling of that grid (zeros outside it) on a 2x output grid of (N + 6) * 2 points per axis with
 * ADA's -0.5 origin shift between the grids, and 2x downsampling with the same taps as a correlation, pads (-1, -1).  Colour after.
 * Domain, per image: finite entries, both singular values of the 2x2 part in [1/16, 16], |translation| <= 64 * max(H, W) in each
 * coordinate; an image outside it is written as NaN (other images are untouched).  One launch on `stream`, no workspace, no host
 * sync, no atomics.  The arguments, parameter rules and errors of gf_augment_nchw, plus GF_ERR_INVALID for a NULL frac. */
int gf_augment_resample_nchw(const float* x, float* y, const int* geom, const float* frac, const float* color, int B, int C, int H, int W,
                             void* stream);

/* The adjoint of gf_augment_resample_nchw's linear part: gx = A^T gy (the colour offset does not take part), gathered per source
 * pixel over the mirrored copies of it that the output can reach, in a fixed order: the same bits on every run and under replay. */
int gf_augment_resample_adjoint_nchw(const float* gy, float* gx, const int* geom, const float* frac, const float* color, int B, int C,
                                     int H, int W, void* stream);

/* ADA's image-space filtering and additive noise (SURVEY A.4 item 17), after the geometry and colour above.  x, y [B, C, H, W]:
 *   gains  float [B, 4] or NULL (no filter): per image the taps h_b = sum_i gains[b][i] bank[i] of the fixed [4, 43] bank (exact
 *          dyadic entries, numerators over 2^15), and y_b = V_b H_b x_b for every channel, (H x)[j] = sum_t h_b[t] x[R_N(j + t - 21)]
 *          along each axis, R_N the mirror of gf_augment_nchw.  An image whose gains are exactly (1, 1, 1, 1) is copied.
 *   sigma  float [B] and noise float [B, C, H, W], both given or both NULL: y_b += sigma_b noise_b; an image with sigma_b == 0 does
 *          not read noise.
 * One launch on `stream`, no workspace, no host sync, no atomics.  Errors, before touching the device: GF_ERR_INVALID for a NULL x / y,
 * only one of sigma and noise, a size <= 0, or y overlapping x; GF_ERR_UNSUPPORTED for H or W < 22 with gains given (one reflection
 * must cover the 21-pixel halo), and H or W > 32768 or C*H*W >= 2^31. */
int gf_augment_filter_nchw(const float* x, float* y, const float* gains, const float* sigma, const float* noise, int B, int C, int H, int W,
                           void* stream);

/* The adjoint of the filter: gx = H_b^T V_b^T gy (the noise does not take part).  Gather only: each source pixel sums its at most
 * 3 preimages per axis under R_N (itself, -m, 2(N-1) - m) in that order, so the result is the same bits on every run and under
 * CUDA-graph replay.  gains is required; otherwise the arguments and errors of gf_augment_filter_nchw. */
int gf_augment_filter_adjoint_nchw(const float* gy, float* gx, const float* gains, int B, int C, int H, int W, void* stream);

/* Image self-attention (img2img, SURVEY A.4 item 18): the n x n part of the layer, per image b and head j, on wgmma (TF32 operands,
 * fp32 accumulation), streamed over 64-token tiles with an online softmax; no n x n tensor is stored (csrc/gf_self_attn.cu).
 * Tensors are channels-last [B, n, C]; head j is the column segment [j d, (j+1) d), h = C / d heads.
 *   O_j = softmax_keys(Q_j K_j^T * scale) V_j,   lse [B, h, n] = log2 sum_keys 2^(Q_j K_j^T * scale * log2 e)  (base-2 units).
 * wgmma reads 32-bit operands along their contraction index only, so the products that contract over tokens take per-head
 * transposed copies instead of the natural tensors: vt = V^T, qt = Q^T, kt = K^T, dOt = dO^T, each [B, C, n] (= [B, h, d, n]).
 * The backward recomputes P from q, k and lse and writes dq, dk, dv [B, n, C]; delta [B, h, n] is scratch it fills with
 * rowsum(dO o O).  Every output element is accumulated by one thread in a fixed order (no atomics): the same bits on every call.
 * Both enqueue on `stream` only: no allocation, no host synchronisation (CUDA-graph capturable).
 * Errors, before the device is touched: GF_ERR_INVALID for a NULL or not 16-byte aligned pointer, a size <= 0, C % d != 0 or a
 * scale that is not positive and finite; GF_ERR_UNSUPPORTED for d not in {32, 64}, n % 64 != 0, B > 65535 or B*n*C >= 2^31. */
int gf_self_attn_fwd(const float* q, const float* k, const float* vt, float* o, float* lse, int B, int n, int C, int d, float scale,
                     void* stream);
int gf_self_attn_bwd(const float* q, const float* qt, const float* k, const float* kt, const float* v, const float* o, const float* lse,
                     const float* dO, const float* dOt, float* delta, float* dq, float* dk, float* dv, int B, int n, int C, int d,
                     float scale, void* stream);

/* The double backward: the vector-Jacobian product of gf_self_attn_bwd as a function (q, k, v, dO) -> (dq, dk, dv), with cotangents
 * a of dq, bk of dk and cv of dv, all [B, n, C].  lse and delta are those of the forward and of gf_self_attn_bwd (delta carries the
 * whole dependence on O).  Writes gq, gk, gv, gdo [B, n, C]; row_r and row_t [B, h, n] are scratch it fills with the row statistics
 * r = rowsum(P o GdS) and t = rowsum(P o GP).  The products that contract over tokens take the per-head transposed copies qt, kt, vt,
 * dOt, at, bkt, cvt [B, C, n].  No n x n tensor is stored; three kernels, each output element accumulated by one thread in a fixed
 * order (no atomics), so the same bits on every call.  Enqueue only, CUDA-graph capturable; the argument rules and errors of
 * gf_self_attn_bwd. */
int gf_self_attn_bwd_vjp(const float* q, const float* qt, const float* k, const float* kt, const float* v, const float* vt, const float* dO,
                         const float* dOt, const float* lse, const float* delta, const float* a, const float* at, const float* bk,
                         const float* bkt, const float* cv, const float* cvt, float* row_r, float* row_t, float* gq, float* gk, float* gv,
                         float* gdo, int B, int n, int C, int d, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GF_OPS_H_ */

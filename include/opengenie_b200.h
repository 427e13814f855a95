/* opengenie_b200.h — C ABI of libopengenie_b200.so (sm_90a only).
 *
 * The drop-in boundary for open-genie's data-parallel hot path. The reference has no FFI of its own:
 * every entry point below replaces one ATen call site (or a fused run of them) in the reference's
 * Python modules; the file:line each one replaces is cited next to its declaration
 * (paths relative to the reference repo, myscience/open-genie @ 732b9f9).
 *
 * Conventions
 *   - plain pointers and sizes only; the caller owns every buffer (device memory) and the stream.
 *   - activations are NDHWC ("channels-last-3d") bf16 unless stated otherwise: x[n][t][h][w][c].
 *   - convolution weights live in "packed" order w[cout][tap][cin] (tap = (it*kh + ih)*kw + iw), which
 *     is exactly the memory order of a torch (Cout,Cin,kt,kh,kw) tensor in channels_last_3d format.
 *   - every function returns OG_OK (0) or a negative og_status; og_last_error() gives the message.
 *     Nothing throws, nothing allocates device memory, nothing synchronises the stream.
 *   - there is NO CPU or library fallback: on a non-sm_90 device the launch fails with OG_ERR_CUDA.
 */
#ifndef OPENGENIE_B200_H_
#define OPENGENIE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum og_status {
  OG_OK = 0,
  OG_ERR_INVALID_ARGUMENT = -1,
  OG_ERR_UNSUPPORTED_SHAPE = -2,
  OG_ERR_CUDA = -3,
} og_status;

typedef void* og_stream_t; /* cudaStream_t */

/* Last error message of the calling thread ("" if none). */
const char* og_last_error(void);
/* Library/ABI version and the SM architecture it was compiled for (100). */
int og_abi_version(void);
int og_compiled_sm(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
uint64_t og_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * conv3d — implicit GEMM on wgmma tensor cores (TMA-staged NDHWC tiles, fp32 accumulate in registers)
 * ---------------------------------------------------------------------------------------------- */

/* Forward 3-D convolution, stride 1, "same" output size, zero padding.
 * Replaces: F.pad + nn.Conv3d in CausalConv3d.forward (genie/module/video.py:178-192) with
 * pad_t_front = kt-1; nn.Conv3d(k=3,p=1) in VideoResidualBlock.main (video.py:609-629) with
 * pad_t_front = 1; the ST-block FFN conv (genie/module/attention.py:429-438, misc.py:94-97);
 * and, through the optional second segment, the always-present 1x1x1 shortcut conv plus the residual
 * add `main(x) + res(x)` (video.py:599-603, 648).
 *
 *   out[n,t,h,w,co] = bias0[co] + bias1[co]
 *                   + sum_{it,ih,iw,ci} x0[n, t+it-pt, h+ih-ph, w+iw-pw, ci] * w[co][(it,ih,iw)][ci]
 *                   + sum_{ci}          x1[n, t, h, w, ci]                  * w[co][kt*kh*kw*c0 + ci]
 *
 * x0: bf16 [N,T,H,W,c0], c0 % 64 == 0.  x1: bf16 [N,T,H,W,c1] or NULL (c1 % 64 == 0).
 * w : bf16 [cout][ldw], ldw >= kt*kh*kw*c0 + c1, ldw % 8 == 0.
 * out: [N,T,H,W,cout], bf16 or fp32 (out_f32 != 0). bias0/bias1: fp32 [cout] or NULL.
 * residual: optional bf16 [N,T,H,W,cout] added in fp32 before the output rounding (the `ffn(x) + x` skip of
 * SpaceTimeAttention, attention.py:472).
 * Reads outside [0,T)x[0,H)x[0,W) are zero (pad_mode='constant').
 * workspace (optional, may be NULL): N*T*H*W*cout fp32 of scratch enables split-K for problems whose tiles
 * cannot fill the 132 SMs (small T*H*W, deep K); without it the same result is computed unsplit. With room for one
 * such slab per split (20 MB always suffices) every split stores its partial tile with plain stores and the finish pass
 * adds the slabs (and emits gn_sums); a smaller workspace is zeroed and reduced into with red.global.add.
 * gn_sums (optional): fp64 [N][2] += (sum, sum of squares) of the bf16 output per sample — the og_gn_stats
 * result for a following GroupNorm(1, C) — produced in the GEMM epilogue when the tiling allows it, otherwise
 * by an internal og_gn_stats pass; either way the caller just zeroes it first. */
/* workspace protocol (og_conv3d_fwd / og_conv3d_dgrad). A workspace PREPARED with og_workspace_init (call it once after
 * allocating the buffer; it zeroes the buffer and reserves its last 4096 bytes for self-resetting counters) enables
 *   - with OG_SPLITK_FUSED=1, the in-kernel split-K finish: the last of a tile's split items to arrive reads the tile's
 *     partial sums back, adds the bias, rounds, stores, emits the GroupNorm sums and re-zeroes its part of the workspace —
 *     no memset, no finish launch, no statistics pass (an experiment: 98 fewer launches per step but 1-1.7 ms slower);
 *   - with OG_IGEMM_DYNAMIC=1, dynamic tile scheduling for the persistent CTAs (an experiment: no measurable gain).
 * An unprepared workspace gets the classic memset + partial sums + finish launch; NULL disables split-K. Results are
 * identical up to the order of fp32 additions. Do not write to a prepared workspace from outside these calls. */
int og_workspace_init(void* workspace, size_t workspace_bytes, og_stream_t stream);

int og_conv3d_fwd(const void* x0, int c0, int kt, int kh, int kw, int pt, int ph, int pw, const void* x1, int c1,
                  const void* w, int ldw, const float* bias0, const float* bias1, const void* residual, void* out,
                  int out_f32, int N, int T, int H, int W, int cout, void* workspace, size_t workspace_bytes,
                  double* gn_sums, og_stream_t stream);

/* Data gradient of the same convolution (autograd's conv3d backward-input, reached from
 * video.py:192 / 609-629 / 599-603 during loss.backward()).
 *   dx[n,t,h,w,ci] = sum_{it,ih,iw,co} dy[n, t-(it-pt), h-(ih-ph), w-(iw-pw), co] * w[co][k_off + tap*cin + ci]
 * dy: bf16 [N,T,H,W,cout] (cout % 64 == 0; a narrower gradient is zero-padded by the caller and
 * w_rows <= cout gives the number of real weight rows); w as above (k_off selects the segment inside
 * a packed row, k_off % 8 == 0); dx: [N,T,H,W,cin] (cin % 64 == 0), bf16 or fp32.
 * red_* (optional): when dx is the gradient of y = act(x*A + B) (a GroupNorm+SiLU fed by this conv's input),
 * red_S[n][c] += (sum_v dpre, sum_v dpre*x) with dpre = dx * act'(x*A+B) — exactly og_affine_act_bwd_reduce on
 * (dx, red_x) — is accumulated in the GEMM epilogue (or by an internal pass when the tiling does not allow it). */
int og_conv3d_dgrad(const void* dy, int cout, int w_rows, const void* w, int ldw, int k_off, int kt, int kh, int kw,
                    int pt, int ph, int pw, void* dx, int dx_f32, int N, int T, int H, int W, int cin,
                    void* workspace, size_t workspace_bytes, const void* red_x, const float* red_A,
                    const float* red_B, int red_act, float* red_S, og_stream_t stream);

/* Weight gradient (autograd's conv3d backward-weight). ACCUMULATES into dw (caller zeroes it):
 *   dw[co][tap][ci] += sum_{n,t,h,w} dy[n,t,h,w,co] * x[n, t+it-pt, h+ih-ph, w+iw-pw, ci]
 * dy: bf16 [N,T,H,W,cout]; x: bf16 [N,T,H,W,cin] (cin % 64 == 0); dw: fp32, row stride ld_dw elements,
 * tap-major / channel-minor inside a row (the channels_last_3d order of the torch weight).
 * workspace (may be NULL): fp32 scratch for the stream-K split over the SMs — up to two 128 x 256 partial tiles
 * (+ 128 bias partials) per SM, added in k order, so the result is the same every run; with less workspace the split
 * shrinks to what fits (whole tiles per CTA without a workspace). */
int og_conv3d_wgrad(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt, int kh,
                    int kw, int pt, int ph, int pw, int N, int T, int H, int W, void* workspace,
                    size_t workspace_bytes, og_stream_t stream);
/* og_conv3d_wgrad + the bias gradient of the same nn.Conv3d in one launch: dbias[c] += sum over voxels of dy[v][c] for
 * c < n_bias (1 <= n_bias <= cout; caller zeroes dbias). The sums come out of the same tensor-core pass (an extra N = 16
 * product against a tile of ones in the tiles that hold the first columns). Replaces the bias half of autograd's conv3d backward
 * (genie/module/video.py:178-192, 609-629). */
int og_conv3d_wgrad_bias(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt, int kh,
                         int kw, int pt, int ph, int pw, int N, int T, int H, int W, float* dbias, int n_bias,
                         void* workspace, size_t workspace_bytes, og_stream_t stream);

/* Strided CausalConv3d — SpaceTimeDownsample (genie/module/video.py:457-483) — as the SAME implicit GEMM, no im2col:
 * geometry of video.py:154-164 (time padded at the FRONT only by pt = (kt-1) + (1-st); space symmetrically by
 * ph = (kh-1)/2, pw = (kw-1)/2), output extents To = (T+pt-kt)/st+1, Ho = (H+2ph-kh)/sh+1, Wo likewise.
 *   fwd  : the A box of a tap is a TMA box with element strides (st,sh,sw); OOB zero fill is the padding.
 *   dgrad: input position i only receives taps == (i+pad) mod s, so the input grid splits into st*sh*sw residue
 *          classes; each is a stride-1 implicit GEMM over dy with its tap subset, stored at stride s into dx
 *          (st*sh*sw launches, no col2im, no atomics).
 *   wgrad: dY boxes on the output grid, x boxes strided on the input grid; ACCUMULATES into dw; workspace as
 *          og_conv3d_wgrad.
 * x / dx: bf16 [N,T,H,W,cin] (cin % 64 == 0); out: [N,To,Ho,Wo,cout]; dy: bf16 [N,To,Ho,Wo,cout] with cout % 64 == 0
 * (zero padded by the caller; w_rows = real weight rows); w: packed bf16 [cout][ldw] as for og_conv3d_fwd. */
int og_conv3d_strided_fwd(const void* x, int cin, int kt, int kh, int kw, int st, int sh, int sw, int pt, int ph, int pw,
                          const void* w, int ldw, const float* bias, void* out, int out_f32, int N, int T, int H, int W,
                          int cout, og_stream_t stream);
int og_conv3d_strided_dgrad(const void* dy, int cout, int w_rows, const void* w, int ldw, int kt, int kh, int kw, int st,
                            int sh, int sw, int pt, int ph, int pw, void* dx, int N, int T, int H, int W, int cin,
                            og_stream_t stream);
int og_conv3d_strided_wgrad(const void* dy, int cout, const void* x, int cin, float* dw, int64_t ld_dw, int kt, int kh,
                            int kw, int st, int sh, int sw, int pt, int ph, int pw, int N, int T, int H, int W,
                            void* workspace, size_t workspace_bytes, og_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm / AdaptiveGroupNorm (+SiLU), NDHWC bf16, HBM-bound passes
 * Replaces F.group_norm / nn.GroupNorm + nn.SiLU (genie/module/video.py:607-608,622-623;
 * tokenizer.py:75-79,163-167; genie/module/misc.py:93) and AdaptiveGroupNorm.forward
 * (genie/module/norm.py:55-69), forward and backward.
 * ---------------------------------------------------------------------------------------------- */

/* sums[n][g] = (sum x, sum x^2) over the group, accumulated in fp64 (caller zeroes sums: N*G*2 doubles).
 * x: bf16 [N,V,C]; C % 8 == 0, (C/G) % 8 == 0, G <= 64. */
int og_gn_stats(const void* x, int N, int64_t V, int C, int G, double* sums, og_stream_t stream);

/* Folds statistics, affine (gamma, beta: fp32 [C] or NULL) and the optional AdaGN modulation
 * (cond_scale, cond_shift: fp32 [N,C] or NULL) into y = x*A[n][c] + B[n][c]; also writes
 * mean_rstd[n][g] = (mean, rstd) for the backward pass. */
int og_gn_finalize(const double* sums, int N, int C, int G, int64_t V, float eps, const float* gamma,
                   const float* beta, const float* cond_scale, const float* cond_shift, float* A, float* B,
                   float* mean_rstd, og_stream_t stream);

/* y = act(x*A + B); act: 0 = identity, 1 = SiLU, 2 = LeakyReLU(0.01) (the discriminators' nn.LeakyReLU(),
 * genie/module/image.py:124-137), 3 = ReLU (VGG16 of the perceptual loss). x,y: bf16 [N,V,C]. The same codes are
 * accepted by every `act` argument below. */
int og_affine_act_fwd(const void* x, const float* A, const float* B, void* y, int N, int64_t V, int C, int act,
                      og_stream_t stream);

/* S[n][c] = (sum_v dpre, sum_v dpre*x), dpre = dy * act'(x*A+B). Caller zeroes S (N*C*2 floats).
 * workspace (may be NULL): fp32 scratch for per-block partial sums, added in block order (reproducible); the number of
 * blocks per sample shrinks to what fits (one per sample without a workspace). */
int og_affine_act_bwd_reduce(const void* dy, const void* x, const float* A, const float* B, int act, float* S,
                             int N, int64_t V, int C, void* workspace, size_t workspace_bytes, og_stream_t stream);

/* Turns S into the per-(n,c) coefficients of dx = A*dpre + Q*x + R and the parameter gradients:
 * dgamma/dbeta [C] are ACCUMULATED (+=); dcond_scale/dcond_shift [N,C] are written. Any of the four may
 * be NULL. */
int og_gn_bwd_finalize(const float* S, const float* mean_rstd, const float* gamma, const float* beta,
                       const float* cond_scale, int N, int C, int G, int64_t V, float* Q, float* R, float* dgamma,
                       float* dbeta, float* dcond_scale, float* dcond_shift, og_stream_t stream);

/* dx = A*dpre + Q*x + R (+ add). Q,R NULL => pure activation backward. add: optional bf16 [N,V,C]. */
int og_affine_act_bwd_apply(const void* dy, const void* x, const float* A, const float* B, const float* Q,
                            const float* R, const void* add, void* dx, int act, int N, int64_t V, int C,
                            og_stream_t stream);

/* AdaptiveGroupNorm conditioning (genie/module/norm.py:58-66): cbar = mean over (t,h,w) of cond [N][V][D] (fp32,
 * channels-last rows), scale = w_scale cbar + b_scale, shift = w_shift cbar + b_shift (the two nn.Linear(dim_cond, C)),
 * all in one launch; the backward launch writes (does not accumulate) dw_* [C][D], db_* [C] and, if dcond != NULL,
 * dcond [N][V][D] = (dscale w_scale + dshift w_shift) / V broadcast over the voxels. D <= 64. */
int og_adagn_cond_fwd(const float* cond, int N, int64_t V, int D, const float* w_scale, const float* b_scale,
                      const float* w_shift, const float* b_shift, int C, float* cbar, float* scale, float* shift,
                      og_stream_t stream);
int og_adagn_cond_bwd(const float* dscale, const float* dshift, const float* cbar, const float* w_scale,
                      const float* w_shift, int N, int64_t V, int D, int C, float* dw_scale, float* db_scale,
                      float* dw_shift, float* db_shift, float* dcond, og_stream_t stream);

/* One-launch forms of the two pairs above, used on the training hot path (same math, same outputs):
 * og_gn_act_fwd  = og_gn_finalize + og_affine_act_fwd  (A, B, mean_rstd are still written for backward);
 * og_gn_act_bwd  = og_gn_bwd_finalize + og_affine_act_bwd_apply, S/mean_rstd NULL => pure activation backward.
 * dx_colsum (optional, float[C], ACCUMULATED) receives sum over rows of dx — the bias gradient of the
 * convolution that produced x (nn.Conv3d bias of ResidualBlock conv #1, genie/module/video.py:609-615); its per-block
 * partials go to the fp32 workspace (at least N*C floats when N > 1) and are added in block order (reproducible).
 * Both need (C/G) % 8 == 0. */
int og_gn_act_fwd(const void* x, const double* sums, const float* gamma, const float* beta, const float* cond_scale,
                  const float* cond_shift, float eps, int G, int act, void* y, float* A, float* B, float* mean_rstd,
                  int N, int64_t V, int C, og_stream_t stream);
int og_gn_act_bwd(const void* dy, const void* x, const float* A, const float* B, const float* S,
                  const float* mean_rstd, const float* gamma, const float* beta, const float* cond_scale, int G, int act,
                  const void* add, void* dx, float* dgamma, float* dbeta, float* dcond_scale, float* dcond_shift,
                  float* dx_colsum, int N, int64_t V, int C, void* workspace, size_t workspace_bytes,
                  og_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * layout / data movement
 * ---------------------------------------------------------------------------------------------- */

/* NCDHW fp32 (the reference's tensor format at every public method, e.g. tokenizer.py:307-330) to the
 * internal NDHWC format (bf16, or fp32 when y_f32) and back. V = T*H*W. */
int og_ncdhw_f32_to_ndhwc(const float* x, void* y, int y_f32, int N, int C, int64_t V, og_stream_t stream);
int og_ndhwc_to_ncdhw_f32(const void* x, int x_f32, float* y, int N, int C, int64_t V, og_stream_t stream);

/* Depth-to-space-time: Rearrange('b (c p q r) t h w -> b c (t p) (h q) (w r)') of
 * DepthToSpaceTimeUpsample (genie/module/video.py:403-408). x: bf16 [N,T,H,W,c*p*q*r] un-shuffled,
 * y: bf16 [N,T*p,H*q,W*r,c] shuffled. inverse=0 reads x writes y; inverse=1 reads y writes x (backward). */
int og_pixel_shuffle3d(const void* x, void* y, int inverse, int N, int T, int H, int W, int c, int p, int q, int r,
                       og_stream_t stream);

/* Explicit im2col for the layers the implicit-GEMM kernel does not take directly: strided
 * CausalConv3d (SpaceTimeDownsample, video.py:477-483) and Cin not a multiple of 64.
 * Causal geometry (video.py:154-164): pt is the FRONT time pad only; ph/pw are symmetric.
 * col: bf16 [N*To*Ho*Wo][kpad], k = tap*C + ci, zero beyond kt*kh*kw*C. col2im is its adjoint. */
int og_im2col3d(const void* x, void* col, int N, int T, int H, int W, int C, int kt, int kh, int kw, int st, int sh,
                int sw, int pt, int ph, int pw, int kpad, og_stream_t stream);
int og_col2im3d(const void* dcol, void* dx, int dx_f32, int N, int T, int H, int W, int C, int kt, int kh, int kw,
                int st, int sh, int sw, int pt, int ph, int pw, int kpad, og_stream_t stream);

/* BlurPooling3d with num_groups == 1 (genie/module/video.py:487-537): every output channel is
 * blur_k(sum_c x[:, c]) with the normalised Pascal kernel, stride (st,sh,sw), padding (k-1)/2.
 * backward == 0: x [N,T,H,W,cin] -> y [N,To,Ho,Wo,cout], scratch >= N*T*H*W floats.
 * backward != 0: x = dy [N,To,Ho,Wo,cout] -> y = dx [N,T,H,W,cin], scratch >= N*To*Ho*Wo floats. */
int og_blurpool3d(const void* x, void* y, float* scratch, int backward, int N, int T, int H, int W, int cin, int cout,
                  int k, int st, int sh, int sw, og_stream_t stream);

/* BlurPooling2d with num_groups == 1 (genie/module/image.py:43-85; registry name 'blur_pool'): x [N,H,W,cin] ->
 * y [N,Ho,Wo,cout], Pascal kernel k x k, stride (sh, sw), symmetric padding `pad` (the reference uses (k-1)//stride). */
int og_blurpool2d(const void* x, void* y, float* scratch, int backward, int N, int H, int W, int cin, int cout, int k,
                  int sh, int sw, int pad, og_stream_t stream);

/* mse_loss (tokenizer.py:364, action.py:166): loss_sum += sum (rec - tgt)^2 ; rec NDHWC fp32, tgt NCDHW fp32.
 * Backward writes gscale * 2 (rec - tgt) / numel as bf16 NDHWC with cpad >= C channels (zero padded) so it
 * can feed og_conv3d_dgrad / og_conv3d_wgrad directly. gscale: device scalar or NULL (= 1). */
int og_mse_fwd(const float* rec_ndhwc, const float* tgt_ncdhw, int N, int C, int64_t V, float* loss_sum,
               og_stream_t stream);
int og_mse_bwd(const float* rec_ndhwc, const float* tgt_ncdhw, const float* gscale, int N, int C, int cpad,
               int64_t V, void* drec, og_stream_t stream);

/* Perceptual-loss pieces that are not convolutions (genie/module/loss.py:34-107, torchvision vgg16.features):
 * nn.MaxPool2d(2, 2) on NHWC bf16 (C % 8 == 0), and out[0] += sum (a - b)^2 over n bf16 elements (n % 8 == 0) — the
 * feature-space mse_loss numerator (loss.py:100-103). The VGG convolutions / ReLUs run on og_conv3d_fwd (kt = 1) and
 * og_affine_act_fwd (act = 3). */
int og_maxpool2x2(const void* x, void* y, int N, int H, int W, int C, og_stream_t stream);
int og_sqdiff_sum(const void* a, const void* b, int64_t n, float* out, og_stream_t stream);

/* out[c] += sum_rows x[row][c] (conv bias gradient). x: bf16 [rows][ld]. */
int og_colsum(const void* x, int64_t rows, int C, int ld, float* out, og_stream_t stream);
/* y[row][0:cd] = x[row][0:cs] zero-padded / truncated; x fp32 or bf16, y bf16. */
int og_pad_channels(const void* x, int x_f32, void* y, int64_t rows, int cs, int cd, og_stream_t stream);

/* out = a - b on n bf16 elements (n % 8 == 0). */
int og_sub_rows(const void* a, const void* b, void* out, int64_t n, og_stream_t stream);

/* dst[row*dst_ld + c] = bf16(src[row*src_ld + c]) for c < cols: refreshes the bf16 operand copy of a
 * conv weight (the cast torch.autocast performs on every conv call, config/tokenize.yaml:78) into one
 * segment of a packed [cout][ldw] weight matrix. src: fp32 or bf16. */
int og_copy_rows_to_bf16(const void* src, int src_f32, int64_t src_ld, void* dst, int64_t dst_ld, int64_t rows,
                         int cols, og_stream_t stream);

/* Data path (genie/module/data.py:181-234, Platformer2D.load_video_slice): decoded frames uint8 [N][T][H][W][3]
 * as cv2.VideoCapture.read() returns them (bgr != 0) -> the colour swap of cvtColor(BGR2RGB), `/ 255.` and the
 * 't h w c -> c t h w' rearrange in one pass on the device, so the host ships 1 byte per element instead of 4.
 * out_kind 0: NCDHW fp32 [N,3,T,H,W]; out_kind 1: NDHWC bf16 with channel pitch cpad >= 3 (zero padded). */
int og_frames_u8_to_video(const uint8_t* frames, int bgr, void* out, int out_kind, int cpad, int N, int T, int H, int W,
                          og_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Lookup-Free Quantization (genie/module/quantization.py:77-133)
 * ---------------------------------------------------------------------------------------------- */
size_t og_lfq_workspace_bytes(int64_t ntok, int D);

/* x: fp32 [ntok][ldx] (first D columns), the tensor AFTER proj_inp / 'b d ... -> b ... d'.
 * out_f32 [ntok][D] and/or out_bf16 [ntok][ld_bf16] (zero padded): sign(x) in eval mode, the straight-
 * through value x + (sign(x) - x) in training mode (line 101). idx: int64 [ntok], MSB-first bit pack (98).
 * training != 0 additionally writes loss[0] =
 *   w_entropy * (mean_n H(p_n) + w_div * H(mean_n p_n)) + w_commit * mse(x, sign x)      (lines 116-131)
 * and fills the workspace (og_lfq_workspace_bytes) that og_lfq_bwd consumes. */
int og_lfq_fwd(const float* x, int ldx, int64_t ntok, int D, float beta, int training, float w_commit,
               float w_entropy, float w_div, float* out_f32, void* out_bf16, int ld_bf16, int64_t* idx, float* loss,
               void* workspace, og_stream_t stream);

/* dx = gloss * dloss/dx + dout (straight-through). gloss: device scalar (NULL = 1); dout: fp32
 * [ntok][ld_dout] or NULL. Writes dx_f32 and/or dx_bf16, both [ntok][ld_dx] with columns >= D zeroed. */
int og_lfq_bwd(const float* x, int ldx, int64_t ntok, int D, float beta, float w_commit, float w_entropy,
               const float* gloss, const float* dout, int ld_dout, float* dx_f32, void* dx_bf16, int ld_dx,
               void* workspace, og_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * factored space-time attention (genie/module/attention.py)
 * All tensors are NDHWC rows [B*T*H*W][C] bf16; a spatial sequence is the H*W rows of one frame, a
 * temporal sequence the T rows of one pixel (stride H*W rows) — no transposition copies.
 * ---------------------------------------------------------------------------------------------- */

/* y = LayerNorm(RoPE(x)): RotaryEmbedding.forward/apply (attention.py:48-94: interleaved pairs over the full
 * channel dim, fp32 angle = pos * freq[i]) followed by nn.LayerNorm (attention.py:219-220).
 * pos(row) = (row / pos_div) % pos_mod — spatial: (1, H*W); temporal: (H*W, T). freq: fp32 [C/2]. */
/* cos_sin (optional, both passes): fp32 [pos_mod][C/2][2] = (cos, sin)(pos * freq[i]) written by og_rope_table — the
 * same sincosf values the passes would otherwise evaluate per element (the '2d' angles reach ~4000 rad: sincosf's slow
 * range reduction made these passes SM-bound at 0.4 of the HBM roofline). Results are bit-identical with and without. */
int og_rope_table(const float* freq, int npos, int C, float* table, og_stream_t stream);
int og_rope_ln_fwd(const void* x, const float* freq, const float* gamma, const float* beta, float eps, void* y,
                   int64_t rows, int C, int64_t pos_div, int pos_mod, const float* cos_sin, og_stream_t stream);
/* dx = RoPE^T(LN'(g0 + g1 + g2)) + add ; dgamma/dbeta accumulated (+=). g1, g2, add may be NULL. */
int og_rope_ln_bwd(const void* x, const float* freq, const float* gamma, float eps, const void* g0, const void* g1,
                   const void* g2, const void* add, void* dx, float* dgamma, float* dbeta, int64_t rows, int C,
                   int64_t pos_div, int pos_mod, const float* cos_sin, og_stream_t stream);

/* Spatial attention: F.scaled_dot_product_attention(q,k,v, scale) non-causal (attention.py:229-234) on
 * wgmma tensor cores. q,k,v,out: [nseq][S][C], C = n_head*64. lse: fp32 [nseq][n_head][S] (saved for backward).
 * residual / out_res (optional, bf16 like out): out_res = out + residual, i.e. `attn(x) + skip(x)`
 * (attention.py:470-471), added in fp32; `out` itself is still written (the backward pass needs it). */
int og_flash_attn_fwd(const void* q, const void* k, const void* v, void* out, const void* residual, void* out_res,
                      float* lse, int nseq, int S, int C, int n_head, float scale, og_stream_t stream);
/* delta_ws: fp32 [nseq][n_head][S] scratch. dq, dk, dv: bf16 [nseq][S][C]. */
int og_flash_attn_bwd(const void* q, const void* k, const void* v, const void* out, const void* dout,
                      const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int nseq, int S, int C,
                      int n_head, float scale, og_stream_t stream);

/* Temporal attention, is_causal=True (attention.py:347-371, 423): one sequence per (batch, pixel), T <= 32.
 * q/out rows ((b*T + t)*P + p); k,v either the same layout (kv_bcast=0) or [B][T][C] shared by all pixels
 * (kv_bcast=1: latent-action conditioning through to_k/to_v, attention.py:127-129,362-363). */
int og_temporal_attn_fwd(const void* q, const void* k, const void* v, const void* residual, void* out, int B, int T,
                         int64_t P, int C, int n_head, float scale, int kv_bcast, og_stream_t stream);
/* kv_bcast=0: dk, dv bf16 like k, v. kv_bcast=1: dk_bcast, dv_bcast fp32 [B][T][C], ACCUMULATED (+=). */
int og_temporal_attn_bwd(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk, void* dv,
                         float* dk_bcast, float* dv_bcast, int B, int T, int64_t P, int C, int n_head, float scale,
                         int kv_bcast, og_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * DynamicsModel rows (genie/dynamics.py)
 * ---------------------------------------------------------------------------------------------- */

/* out[row] = bf16(tok_w[tok[row]] + act_w[act[row / rows_per_act]]): tok_emb(tokens) + act_emb(act_id) broadcast
 * over (h, w) (dynamics.py:34-38, 55). tok: int64 [rows]; act: int64 [rows / rows_per_act]; weights fp32. */
int og_embed_add_fwd(const int64_t* tok, const int64_t* act, const float* tok_w, const float* act_w, void* out,
                     int64_t rows, int64_t rows_per_act, int C, int tok_vocab, int act_vocab, og_stream_t stream);
/* d_tok_w / d_act_w (fp32, ACCUMULATED): scatter-add of dy (bf16 [rows][C]). */
int og_embed_add_bwd(const int64_t* tok, const int64_t* act, const void* dy, float* d_tok_w, float* d_act_w,
                     int64_t rows, int64_t rows_per_act, int C, int tok_vocab, int act_vocab, og_stream_t stream);

/* cross_entropy(logits[mask], target[mask]) (dynamics.py:89-97). logits bf16 [rows][V]; mask uint8 [rows];
 * row_lse fp32 [rows] (scratch, kept for backward); stats fp32 [2] zeroed by the caller: += (sum loss, count).
 * Backward: dlogits = gloss / count * (softmax - onehot) on masked rows, 0 elsewhere (bf16 [rows][V]). */
int og_masked_ce_fwd(const void* logits, const int64_t* target, const uint8_t* mask, int64_t rows, int V,
                     float* row_lse, float* stats, og_stream_t stream);
int og_masked_ce_bwd(const void* logits, const int64_t* target, const uint8_t* mask, const float* row_lse,
                     const float* stats, const float* gloss, void* dlogits, int64_t rows, int V, og_stream_t stream);

/* MaskGIT iterative sampling — DynamicsModel.generate (genie/dynamics.py:101-165). The reference packs the
 * transformer input once before its loop and never updates it (lines 128-134), so all iterations share one set of
 * logits: og_softmax_cdf turns them into per-position CDFs (softmax(logits / temp), line 143) once, and
 * og_maskgit_sample runs EVERY iteration of lines 136-163 in one launch (one CTA per batch row): inverse-CDF draw with
 * the supplied uniforms (torch.multinomial's role, line 145) -> confidence = prob[pred] (146) -> -inf on already
 * predicted positions (151) -> top-k of `schedule[s]` (152) -> scatter into code / mask (159-160).
 * logits: [rows = B*P][V] bf16 or fp32; cdf: fp32 [rows][V]; uniforms: fp32 [steps][B][P] in [0,1);
 * schedule: int32 [steps] (device); code: int64 [B][P] in/out (initialised to masked_tok); mask: uint8 [B][P] in/out
 * (1 = still to predict). P <= 4096. */
int og_softmax_cdf(const void* logits, int logits_f32, int64_t rows, int V, float inv_temp, float* cdf,
                   og_stream_t stream);
int og_maskgit_sample(const float* cdf, const float* uniforms, const int* schedule, int steps, int B, int P, int V,
                      int64_t* code, uint8_t* mask, og_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * fused multi-tensor AdamW (genie/tokenizer.py:437-442) + bf16 operand refresh
 * ---------------------------------------------------------------------------------------------- */
typedef struct og_adamw_tensor {
  float* p;        /* fp32 master weights, n elements */
  const float* g;  /* fp32 gradient or NULL (then only the bf16 copy is refreshed) */
  float* m;        /* exp_avg */
  float* v;        /* exp_avg_sq */
  void* p_bf16;    /* optional bf16 destination: element i -> [(i / row_len) * dst_ld + i % row_len] */
  int64_t n;
  int64_t row_len;
  int64_t dst_ld;
} og_adamw_tensor;

int og_adamw_chunk_elems(void);
/* table_dev: device array of tensors; chunk_tensor_dev / chunk_index_dev: for every chunk of
 * og_adamw_chunk_elems() elements, which tensor and which chunk inside it. step >= 1.
 * grad_scale_dev: optional device scalar multiplied into every gradient (e.g. 1/world_size). */
/* step_dev / lr_dev (optional): step count and learning rate read from device memory instead of the
 * host arguments, so a CUDA graph that captured the whole training step stays valid across replays;
 * og_adamw_tick increments the device-side step counter (launch it before og_adamw_step). */
int og_adamw_step(const og_adamw_tensor* table_dev, const int* chunk_tensor_dev, const int* chunk_index_dev,
                  int num_chunks, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                  const int* step_dev, const float* lr_dev, const float* grad_scale_dev, og_stream_t stream);
int og_adamw_tick(int* step_dev, og_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* OPENGENIE_B200_H_ */

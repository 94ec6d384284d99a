/* stp3_b200 — C ABI of the H100-native (sm_90a) ST-P3 camera->BEV perception hot path.
 *
 * The reference (OpenDriveLab/ST-P3) is 100 % Python/PyTorch and has no FFI of its own; the drop-in boundary is
 * the nn.Module surface (SURVEY.md §8b).  This header is the C boundary that sits directly underneath those
 * modules: each entry point names the reference interface it replaces (file:line in OpenDriveLab/ST-P3).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch's caching allocator in practice), unless the
 *     parameter is documented as a host value;
 *   - no entry point allocates, frees or synchronises: work is enqueued on `stream` (a cudaStream_t passed as
 *     void*) and the call returns immediately;
 *   - return value: 0 on success, a negative STP3_E* code otherwise; stp3_last_error() returns the text for the
 *     calling thread;
 *   - re-entrant; no global mutable state apart from the thread-local error string.
 */
#ifndef STP3_B200_H_
#define STP3_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STP3_OK 0
#define STP3_EINVAL (-1)   /* bad argument (shape, alignment, null pointer) */
#define STP3_ENOSPC (-2)   /* workspace too small */
#define STP3_ECUDA (-3)    /* CUDA runtime / driver error (launch failure, no device) */
#define STP3_EUNSUPPORTED (-4)

/* Library / build identification ("sm_90a", ABI version). */
int stp3_abi_version(void);
const char* stp3_build_info(void);
const char* stp3_last_error(void);

/* ---------------------------------------------------------------------------------------------------------
 * Lift-splat: softmax(depth) (x) context outer product, ego-motion aligned voxel pooling, temporal discount.
 *
 * Replaces, fused into one scatter kernel + one finalize kernel:
 *   STP3.get_geometry                      stp3/models/stp3.py:186-201   (frustum -> ego points)
 *   STP3.encoder_forward (softmax, outer)  stp3/models/stp3.py:214-221   (never materialised)
 *   STP3.projection_to_birds_eye_view      stp3/models/stp3.py:226-301   (ego warp, voxel index, mask, pooling,
 *                                                                          discount recurrence, (C,X,Y) layout)
 *   VoxelsSumming.forward                  stp3/utils/geometry.py:299-318
 *
 * stp3_lift_splat_desc describes the call: the camera / ego-motion / frustum geometry, the BEV grid, the shapes and the
 * frame range.  The forward and the backward take the same descriptor and their tensors as arguments.
 *
 * Layouts (all fp32 unless noted)
 *   feat          feat_layout==0: (B,S,N,C,Hf,Wf)  [the reference Encoder's NCHW output]
 *                 feat_layout==1: (B,S,N,Hf,Wf,C)  [channels-last, produced by this library's conv kernels]
 *   depth_logits  (B,S,N,D,Hf,Wf); ignored (may be NULL) when use_depth_distribution==0 (stp3.py:218)
 *   cam_M         (B,S,N,3,3) = R . K^-1   evaluated on the host with the reference's torch calls
 *   cam_t         (B,S,N,3)
 *   ego_R, ego_t  (B,S,3,3), (B,S,3)  from pose_vec2mat(future_egomotion)  (geometry.py:158-172)
 *   xs, ys, ds    (Wf), (Hf), (D): the three axes of STP3.create_frustum (stp3.py:111-130)
 *   bev_off       (bev_start_position - bev_resolution/2) as evaluated in fp32 by torch (stp3.py:288)
 *   bev_res       bev_resolution; nx, ny, nz = bev_dimension
 *   ranks_out     optional (B,S,N,D,Hf,Wf) int32: pillar rank ix*(ny*nz)+iy*nz+iz of every lifted point after the
 *                 ego warp, -1 where the reference's mask (stp3.py:239-246) drops it.  Bit-exact with the CPU
 *                 reference; used by the parity tests.
 *   out           out_layout==0: (B,S,C,nx,ny) fp32  [what projection_to_birds_eye_view returns]
 *                 out_layout==1: (B,S,nx,ny,C) fp32  [channels-last]
 *                 out_layout==2: two bf16 planes [2][B,S,nx,ny,C] (hi then lo; C % 8 == 0): the activation format
 *                                of the tensor-core path, consumed directly by stp3_conv_fwd
 *   pool_sum      optional (B,S,C) fp32: sum over the nx*ny cells of out[b,t,c] (feeds the pyramid-pooling branch
 *                 of TemporalBlock, temporal.py:408-423); fully overwritten by the call.
 *   workspace     >= stp3_lift_splat_workspace_bytes(desc) bytes, 256-byte aligned.  It holds the channels-last
 *                 fp32 scatter grid (B,S,nx*ny,C) and a per-pillar occupancy map.  It must be ALL ZERO on entry:
 *                 clear it once with stp3_lift_splat_workspace_init() after allocating it; every successful
 *                 stp3_lift_splat_fwd leaves it zero again (the finalize kernel re-zeroes exactly the pillars it
 *                 read), so no per-call memset is needed.  After a failed call, re-initialise it.
 * nz must be 1 (the reference's squeeze(0) at stp3.py:298 assumes it).
 *
 * Frame-sharded mode (f_count > 0; latency mode, SURVEY.md §8e): when the global batch is smaller than the number of
 * GPUs the B*S camera frames are split across ranks.  Each rank splats its flat frames f_begin + [0, f_count)
 * (f = b*S + t, the ego-motion chain of frame t still uses the poses t..S-2 of its sample) and writes them RAW -- no
 * discount recurrence, `discount` is ignored -- as channels-last fp32 grids (f_count, nx, ny, C): out_layout must be 1
 * and ranks_out and pool_sum NULL.  The workspace is sized for the f_count frames.
 *   n_peers == 0  the frames go to `out`; after ONE all-gather of those grids (ncclAllGather over NVLink;
 *                 stp3_b200/parallel.py) every rank holds (B, S, nx, ny, C) and stp3_bev_discount applies
 *                 out[t] = out[t-1]*discount + raw[t] (stp3.py:296) and emits the bf16 hi/lo planes the temporal block
 *                 consumes.
 *   n_peers > 0   FUSED WITH THE ALL-GATHER (needs C in {32, 64, 128}; `out` is ignored): the finalize epilogue stores
 *                 every finished BEV row of flat frame f straight into slot f of all n_peers gathered buffers
 *                 peer_out[r] (each (B*S, nx, ny, C) fp32, 32-byte aligned; peer-mapped device pointers of every rank's
 *                 buffer including this rank's own, e.g. from CUDA IPC / torch symmetric memory) over NVLink -- no
 *                 separate collective launch.  The caller brackets the call with a cross-rank barrier on both sides
 *                 (buffers free / stores landed) and then runs stp3_bev_discount on its own buffer.  peer_out is a HOST
 *                 array of n_peers <= 8 pointers.
 */
typedef struct stp3_lift_splat_desc {
  const float* cam_M;
  const float* cam_t;
  const float* ego_R;
  const float* ego_t;
  const float* xs;
  const float* ys;
  const float* ds;
  float bev_off[3];
  float bev_res[3];
  int nx, ny, nz;
  float discount;
  int B, S, N, D, Hf, Wf, C;
  int feat_layout;
  int use_depth_distribution;
  int f_begin, f_count;  /* 0, 0: every frame, with the discount recurrence; f_count > 0: frame-sharded mode */
} stp3_lift_splat_desc;

size_t stp3_lift_splat_workspace_bytes(const stp3_lift_splat_desc* desc);
int stp3_lift_splat_workspace_init(void* workspace, size_t workspace_bytes, void* stream);
int stp3_lift_splat_fwd(const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits,
                        int32_t* ranks_out, float* pool_sum, void* workspace, size_t workspace_bytes,
                        float* out, int out_layout, int n_peers, void* const* peer_out, void* stream);

/* The kernels stp3_lift_splat_fwd would launch for these arguments; stp3_lift_splat_fwd launches exactly this plan.
 * Host only: launches nothing and never dereferences feat or depth_logits (their addresses decide the alignment rule
 * and are encoded into the TMA descriptors).  Refuses what stp3_lift_splat_fwd refuses for the descriptor, out_layout
 * and n_peers, with the same messages.
 *   tma_rules       the TMA-staged scatter kernel is admissible: TW 4, Wf % 4 == 0, C % 64 == 0, D <= 256, Hf <= 32,
 *                   16-byte aligned feat / depth_logits, its tile fits in shared memory, STP3_LIFT_NO_TMA unset or 0
 *   scatter         1: the TMA-staged kernel runs (tma_rules and the driver encoded both tensor maps); 0: the generic one
 *   scatter_tw      image columns per generic scatter CTA (4, 2 or 1; 4 whenever tma_rules holds)
 *   finalize        0: lane-per-pillar kernel; 1: channels-last kernel (out_layout != 0, C in {32, 64, 128}, <= 4 frames)
 *   finalize_vec    lane-per-pillar kernel with 8-channel vector accesses (C % 8 == 0); 0 for the channels-last kernel
 *   finalize_smax   frames the finalize kernel is instantiated for (4 or 8)
 *   finalize_lpp    channels-last kernel: lanes per pillar, C / 16 (2, 4 or 8); 0 for the lane-per-pillar kernel
 *   channel_groups  finalize CTAs per pillar block; > 1 (C > 64, lane-per-pillar) adds the occupancy-clearing kernel */
typedef struct stp3_lift_splat_kernel_plan {
  int tma_rules;
  int scatter;
  int scatter_tw;
  int finalize;
  int finalize_vec;
  int finalize_smax;
  int finalize_lpp;
  int channel_groups;
} stp3_lift_splat_kernel_plan;
int stp3_lift_splat_plan(const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits, int out_layout,
                         int n_peers, stp3_lift_splat_kernel_plan* plan);

/* Deterministic form of stp3_lift_splat_fwd (torch.use_deterministic_algorithms; DESIGN.md §3.14).  Same arguments,
 * rules, frame-sharded and peer modes, and the scatter and finalize kernels stp3_lift_splat_plan reports, in their
 * 64-bit fixed-point form:
 *   - a pre-pass finds m_f, the largest finite |feature| of every frame f (all cameras and channels);
 *   - every flushed fp32 partial of frame f is rounded to a multiple of 2^-k_f, k_f = 62 - (ceil(log2 m_f) +
 *     ceil(log2(N*D*Hf*Wf))) (0 for an all-zero frame), and added as int64 (red.global.add.u64).  Probabilities are
 *     <= 1, so no pillar sum reaches 2^63; integer addition is associative, so the sum does not depend on the order in
 *     which CTAs and warps arrive;
 *   - the finalize converts each int64 v to fp32 as __double2float_rn((double)v * 2^-k_f), then runs the unchanged
 *     discount recurrence, hi/lo split and pool partials; the pool slices are added in a fixed order.
 * Result: bitwise identical for the same inputs, build and GPU model.  A frame's values depend on that frame's inputs
 * only (and, through the recurrence, on the earlier frames of its sample): not on the batch it sits in, on
 * f_begin / f_count, or on the rank that computed it.  Within one fp32 ulp of the exact sum of the grid-rounded
 * partials; the rounding adds at most 2^-(k_f+1) per partial.
 * Non-finite values: a NaN or +-inf partial marks its pillar in a per-frame poison bitmap instead of being added; the
 * finalize writes NaN into EVERY channel of a poisoned pillar in that frame, and the recurrence carries it into later
 * frames.  Per-channel fidelity is given up on purpose: a loss scaler only needs to see the NaN.  Non-finite features
 * are left out of m_f.
 * Memory: the int64 grid is twice the fp32 one (perceive at B = 4: 246 MB instead of 123 MB; B = 8, S = 5, 400 x 400,
 * C = 128: 6.6 GB instead of 3.3 GB).  The workspace holds >= stp3_lift_splat_det_workspace_bytes(desc) bytes, which
 * is never less than stp3_lift_splat_workspace_bytes(desc); it obeys the same all-zero rule, so one zeroed workspace
 * serves both entry points, in any interleaving. */
size_t stp3_lift_splat_det_workspace_bytes(const stp3_lift_splat_desc* desc);
int stp3_lift_splat_fwd_det(const stp3_lift_splat_desc* desc, const float* feat, const float* depth_logits,
                            int32_t* ranks_out, float* pool_sum, void* workspace, size_t workspace_bytes,
                            float* out, int out_layout, int n_peers, void* const* peer_out, void* stream);

/* Backward of stp3_lift_splat_fwd (training through the drop-in, SURVEY.md row f2): given grad_out = dLoss/d out
 * (B,S,C,nx,ny) fp32 it returns grad_feat (B,S,N,C,Hf,Wf) and grad_depth_logits (B,S,N,D,Hf,Wf; may be NULL, and is not
 * written when use_depth_distribution == 0).  Replaces the autograd chain of the reference:
 *   VoxelsSumming.backward                 stp3/utils/geometry.py:321-330  (every point receives its pillar's gradient)
 *   projection_to_birds_eye_view           stp3/models/stp3.py:239-296     (mask, index_put, bev = bev*discount + tmp)
 *   outer product + softmax over depth     stp3/models/stp3.py:214-216
 * Voxel indices are recomputed with the forward's exact arithmetic (not differentiable, like the reference's .long()).
 * feat is NCHW (desc->feat_layout 0) and every frame is processed (desc->f_count 0).  scratch:
 * stp3_lift_splat_bwd_scratch_bytes(desc) bytes of device memory (no invariant).  Gathers only, no atomics: deterministic. */
size_t stp3_lift_splat_bwd_scratch_bytes(const stp3_lift_splat_desc* desc);
int stp3_lift_splat_bwd(const stp3_lift_splat_desc* desc, const float* grad_out, const float* feat,
                        const float* depth_logits, void* scratch, size_t scratch_bytes, float* grad_feat,
                        float* grad_depth_logits, void* stream);
/* stp3_lift_splat_bwd for channels-last context features, the layout the encoder heads hand to stp3_lift_splat_fwd
 * (desc->feat_layout 1, required): feat and grad_feat are (B,S,N,Hf,Wf,C), 8-byte aligned, C even; depth_logits and
 * grad_depth_logits stay (B,S,N,D,Hf,Wf).  Same descriptor rules, scratch query and kernels; only the addresses of feat
 * and grad_feat differ (a lane's channel pair is one float2 of a pixel's row), and every sum keeps its order: the
 * results equal stp3_lift_splat_bwd's on the transposed tensors bit for bit. */
int stp3_lift_splat_bwd_cl(const stp3_lift_splat_desc* desc, const float* grad_out, const float* feat,
                           const float* depth_logits, void* scratch, size_t scratch_bytes, float* grad_feat,
                           float* grad_depth_logits, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Dense layers: implicit-GEMM convolution on the Hopper tensor cores (wgmma, register accumulators, TMA-fed operands).
 *
 * One entry point covers every convolution of the temporal block, the per-frame DeepLab head and the BEV decoder:
 *   CausalConv3d / conv_1x1x1_norm_activated / TemporalBlock   stp3/layers/temporal.py:252-273, 315-325, 426-489
 *   ASPP / DeepLabHead / UpsamplingAdd / UpsamplingConcat      stp3/layers/convolutions.py:183-280
 *   Decoder (ResNet-18 stages + heads)                         stp3/models/decoder.py:8-140
 * Eval-mode BatchNorm is folded into w / bias by the caller (stp3_b200/dense.py); ReLU, residual add, per-image
 * bias (the spatially constant pyramid-pool / ASPP-pool / ego-motion branches) and the concat offset are fused.
 *
 * Activations are channels-last and carried as TWO bf16 planes (hi = bf16(x), lo = bf16(x - hi)) so that the bf16
 * tensor pipe reproduces fp32 convolution to ~1e-5 (three MMAs per product: hi*hi + hi*lo + lo*hi):
 *   x_hi, x_lo   (B, T, H, W, in_cstride) bf16, in_cstride % 64 == 0, padding channels zero
 *   w            [ntaps][cin/64][2 planes][bn][64] bf16: tap-major, K-major rows of 64 input channels
 *   bias         [bn] fp32;  img_bias  optional [B*T][bn] fp32: per-image bias table that REPLACES bias (it must
 *                already contain it): the spatially constant branches and the ego-motion channels enter here
 *   res_hi/lo    optional residual (B*T, Ho, Wo, res_cstride), channels [res_coff, res_coff+bn)
 *   y_hi, y_lo   optional output planes (B*T, Ho, Wo, out_cstride), channels [out_coff, out_coff+bn)
 *   y_f32        optional (B*T, n_valid, Ho, Wo) fp32 in the reference's NCHW layout (final logits), or channels-last
 *                (desc.f32_layout = 1)
 * taps[i] = (dt, dy, dx): input coordinate = output coordinate * stride + d (dt is not strided); coordinates
 * outside the tensor read as zero (this is the reference's zero / causal padding).
 */
typedef struct stp3_conv_desc {
  int B, T, H, W;        /* B samples x T frames are processed; the input tensor is (B, T_total, H, W, in_cstride) */
  int T_total, t0;       /* frames [t0, t0+T) of each sample are processed (T_total = 0 means T_total = T, t0 = 0);
                            outputs / residual / img_bias are indexed by the B*T processed images */
  int in_cstride;        /* channels of the input tensor */
  int cin_off, cin;      /* channel window this convolution reads (multiples of 64) */
  int Ho, Wo;            /* output spatial size */
  int stride;            /* spatial stride, 1 or 2 */
  int ntaps;             /* 1 .. 49 */
  signed char taps[49][3];
  int bn;                /* padded output channels: 64, 128 or 256 */
  int out_cstride, out_coff;
  int n_store;           /* output channels actually stored to y_hi/y_lo (multiple of 8, 0 = bn): lets several
                            convolutions write adjacent windows of one concat tensor */
  int relu;              /* apply ReLU */
  int res_mode;          /* 0 none, 1 residual added before the activation, 2 after it */
  int res_cstride, res_coff;
  int n_valid;           /* real output channels written to y_f32 */
  int sigmoid;           /* apply a sigmoid to y_f32 (instance_center head, decoder.py:70) */
  int tune_n_sub;        /* accepted and ignored: the CTA tile is always 8x16 pixels */
  int tune_group;        /* 0 = automatic; 1 = never share an activation load between the dy taps of a 3x3; 3 = share;
                            +4 = stream the weights through the smem ring even if they would fit (more activation stages);
                            +8 = (64-column blocks) one stacked [W_hi; W_lo] operand: 2 MMAs per product instead of 3 */
  int n_cols;            /* output columns that carry weights (0 = bn): rows [n_cols, bn) of every weight block and the
                            bias are zero padding, so the kernel neither loads nor multiplies them (bn <= 128) */
  /* optional (bn = 64): col_sums[img][c] = sum over the output pixels of the activated output (fp32, (B*T, 64)) -- the
     spatial sums the next block's pooling branches need, produced by the epilogue instead of a separate pass.
     col_sums_scratch: stp3_conv_col_sums_scratch_bytes(B*T, 64) bytes of device scratch. */
  float* col_sums;
  float* col_sums_scratch;
  size_t col_sums_scratch_bytes;
  /* optional second destination (bn = 128, plain hi/lo outputs, n_store <= 64): output columns [64, 64 + n_store2) are
     written to y2 (channels [out2_coff, out2_coff + n_store2)) with activation relu2, columns [0, n_store) to y with
     `relu` -- two 64-column convolutions of the same input as ONE launch that reads the input once. */
  void* y2_hi;
  void* y2_lo;
  int out2_cstride, out2_coff, n_store2, relu2;
  /* input channels [k_lo, k_hi) of the window carry data (multiples of 16; k_hi = 0: the whole window): the weights of
     the other channels are zero, so their UMMA K steps are not issued.  k_lo must lie in the first 64-channel block and
     k_hi in the last (narrow convolutions: 35 -> 35 channels of temporal.py:436-461 run 3 of 4 K steps, 32 -> 32 run 2). */
  int k_lo, k_hi;
  int f32_layout;        /* layout of y_f32: 0 = (B*T, n_valid, Ho, Wo) like the reference, 1 = channels-last (B*T, Ho, Wo,
                            n_valid) -- what stp3_lift_splat_fwd(feat_layout = 1) fetches as ONE TMA box per tile (the encoder
                            heads hand their context features over this way, encoder.py:88-95 -> stp3.py:216) */
  int swish;             /* apply swish x * sigmoid(x) to y_hi / y_lo instead of ReLU (EfficientNet expand convolutions);
                            not with relu or a second destination */
  long long w_img_stride; /* 0: one weight tensor for every image; > 0: image i's weights start at w + i * w_img_stride
                            (bf16 elements, a multiple of 64) -- the squeeze-excite gated projections (stp3_se_gate).  Such
                            weights are streamed through the shared-memory ring, never resident */
  int tune_bn;           /* column-block width: 0 = automatic (bn up to 128 in one block, 256 as two of 128), 64 or 128
                            (<= bn).  A convolution of several blocks is ONE launch whose work items are (pixel tile,
                            column block) pairs: more and smaller items for the layers with few tiles, and at 64 the
                            stacked operand (tune_group +8) and deeper shared-memory rings.  Its weights are streamed.
                            Not with a fused head, a second destination or col_sums: they need every column in one CTA */
} stp3_conv_desc;

/* Optional fused 1x1 "head" evaluated on the activated output tile while it is still in registers:
 *   out_k[img, y, x] = b[k] + sum_c w[k][c] * y[img, y, x, c]      (k < n_out <= 8; sigmoid where the mask bit is set)
 * This is the 3x3 conv -> BN -> ReLU -> 1x1 conv(+bias) tail of every decoder head (decoder.py:38-89); several heads
 * that share their input run as ONE convolution (their 3x3 kernels concatenated along N) and each head's 1x1 weights
 * occupy its column block of w.  out[k] points at the (Ho, Wo) fp32 plane of output k for image 0 and consecutive
 * images are img_stride[k] elements apart, so every head writes its own contiguous (n_img, k_out, Ho, Wo) tensor. */
typedef struct stp3_conv_head {
  int n_out;
  const float* w;          /* [n_out][bn] fp32 (device) */
  const float* b;          /* [n_out] fp32 (device) */
  float* out[8];
  long long img_stride[8];
  int sigmoid_mask;
} stp3_conv_head;

/* bytes of device scratch stp3_conv_desc.col_sums needs for n_img images */
size_t stp3_conv_col_sums_scratch_bytes(int n_img, int bn);
/* How stp3_conv_fwd would run desc on a device of n_sm SMs, from the descriptor alone (host arithmetic, no device):
 * work items = tiles of 8x16 pixels x column blocks, walked by `ctas` persistent CTAs; the shared-memory ring depths
 * (b_stages = 0 and resident = 1: the weights stay in shared memory).  Same argument errors as stp3_conv_fwd. */
typedef struct stp3_conv_tiling_info {
  int bn_blk, stacked;
  int tiles, items, ctas;
  int a_stages, b_stages, resident;
} stp3_conv_tiling_info;
int stp3_conv_tiling(const stp3_conv_desc* desc, int n_sm, stp3_conv_tiling_info* out);
int stp3_conv_fwd(const stp3_conv_desc* desc, const void* x_hi, const void* x_lo, const void* w, const float* bias,
                  const float* img_bias, const void* res_hi, const void* res_lo, void* y_hi, void* y_lo,
                  float* y_f32, const stp3_conv_head* head /* may be NULL */, void* stream);

/* Operand kinds of the train-mode convolutions.  HILO: fp32 carried as bf16 hi/lo planes, three MMAs per product (what
 * stp3_conv_fwd, stp3_conv_wgrad and stp3_conv3d_wgrad do).  BF16 / F16: ONE 16-bit plane per operand and one MMA per
 * product, fp32 accumulation -- the convolutions of a training step under torch.autocast(dtype=torch.bfloat16 /
 * torch.float16).  Every fp32 -> 16-bit conversion of this library rounds to nearest even, overflows to +-inf and
 * passes NaN through; nothing saturates, so a loss scaler sees an overflowed gradient as inf / NaN. */
#define STP3_OPERAND_HILO 0
#define STP3_OPERAND_BF16 1
#define STP3_OPERAND_F16 2
/* stp3_conv_fwd with one-plane operands (operand BF16 or F16): x (B, T_total, H, W, in_cstride) is one plane of that
 * kind (padding channels zero) and w is [ntaps][cin/64][bn][64] of the same kind (one plane instead of two per K block).
 * Each K step issues one MMA; the stacked operand (tune_group +8) does not apply and is ignored.  Output: y_f32 only
 * (required), with n_valid / f32_layout / sigmoid and the optional img_bias as in stp3_conv_fwd.  The descriptor rules
 * of stp3_conv_fwd hold, and it must carry no residual, second destination, col_sums, swish or per-image weights. */
int stp3_conv_fwd_plane(const stp3_conv_desc* desc, int operand, const void* x, const void* w, const float* bias,
                        const float* img_bias, float* y_f32, void* stream);
/* stp3_conv_tiling for an operand kind: how stp3_conv_fwd (HILO) or stp3_conv_fwd_plane (BF16 / F16) would run desc.
 * A one-plane operand halves the activation stage and the weight tile, so it may keep weights resident or pick ring
 * depths that the hi/lo pair does not, and it never stacks.  operand HILO answers exactly as stp3_conv_tiling. */
int stp3_conv_tiling_op(const stp3_conv_desc* desc, int n_sm, int operand, stp3_conv_tiling_info* out);

/* ---------------------------------------------------------------------------------------------------------
 * ASPP branches + projection of a DeepLabHead as ONE back-to-back tensor-core kernel (stp3/layers/convolutions.py:242-270):
 *   y = relu(BN(project.0(cat_b relu(BN(conv_b(x))))))   for the spatial branches b (1x1 and the dilated 3x3s); the
 * global-pool branch is spatially constant and enters through img_bias like in stp3_conv_fwd.  The 4 x 128-channel concat
 * tensor never exists: every branch's activated 16x16x128 tile is converted to bf16 hi/lo planes in shared memory and
 * multiplied with its slice of the projection weights while the next branch's convolution runs.  hidden = 128 channels.
 *   x_hi, x_lo  (B, T, H, W, in_cstride) bf16 planes, channels [0, cin) read
 *   w           bf16 rows of 64 (K-major), blocks of [hi: 128 rows][lo: 128 rows]:
 *               first one block per (tap of branch 0.., K block of cin) -- BN folded, rows = hidden channels --
 *               then two per branch for the projection (rows = output channels, K = the branch's hidden channels 0..63, 64..127)
 *   br_bias     [n_br][128] fp32 folded BN shifts of the branches;  img_bias [B*T][128] fp32 projection bias table
 *   y_hi, y_lo  (B*T, H, W, out_cstride) bf16 planes, channels [out_coff, out_coff + 128) written
 */
typedef struct stp3_aspp_desc {
  int B, T, H, W;
  int in_cstride, cin;
  int n_br;                   /* 1 .. 4 spatial branches */
  int n_taps[4];              /* 1 .. 9 each; every branch must contain its centre tap (0, 0) */
  signed char taps[4][9][2];  /* (dy, dx) input offsets */
  int out_cstride, out_coff;
  int no_relu;                /* 0: ReLU on the projection output (ASPP); 1: none (3x3 conv -> 1x1 classifier tail) */
  int n_store;                /* output channels written: 128 (0 = default) or 64 (projection rows 64.. are zero padding) */
} stp3_aspp_desc;
int stp3_aspp_fused_fwd(const stp3_aspp_desc* desc, const void* x_hi, const void* x_lo, const void* w,
                        const float* br_bias, const float* img_bias, void* y_hi, void* y_lo, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Tail of a TemporalBlock (stp3/layers/temporal.py:426-489) as ONE back-to-back tensor-core kernel:
 *   out = relu(BN(aggregation 1x1x1 of [path 0 | path 1 | path 2 | pyramid pooling])) + (projection(x) | x)
 * with path 0 / 1 = the causal (2,3,3) / (1,3,3) convolutions of the entry convolutions' outputs `mid` and path 2 = a
 * 1x1x1 convolution of x.  Up to three MMA chains accumulate the paths side by side (register accumulators), the activated concat is
 * converted to bf16 hi/lo in shared memory and multiplied with the aggregation weights; the 128-channel concat tensor
 * never exists.  Applicable when every path has <= 48 channels, x <= 64 spatial channels and the block <= 64 outputs.
 *   chain: src (0 = mid, 1 = x), cin_off (64-channel K block read), taps (dt, dy, dx), n_mma (MMA width, multiple of 16),
 *          tmem_col (column of its first output in the hidden accumulator, multiple of 16), [k_lo, k_hi) channels with data
 *   piece_col[pp]: hidden-accumulator column of the 8-channel piece pp of the 128-channel operand P (-1 = zeros)
 *   w: bf16 rows of 64, blocks of [hi: 128 rows][lo: 128 rows]; one block per tap of chain 0, 1, 2, then two blocks of the
 *      aggregation weights (K blocks of P), then one of the projection; output channel n of an N-wide chain sits in row
 *      n (n < N/2) or 64 + n - N/2
 *   hid_bias [B*T][128] (P order), img_bias [B*T][64] (aggregation bias + pooling branch), res_bias [B*T][64] or NULL
 *   col_sums optional (B*T, 64): per-image sums over pixels of the output; scratch: stp3_block_fused_scratch_bytes(B*T)
 */
typedef struct stp3_block_chain {
  int src, cin_off, n_taps;
  signed char taps[18][3];
  int n_mma, tmem_col, k_lo, k_hi;
} stp3_block_chain;
typedef struct stp3_block_desc {
  int B, T, H, W;
  int mid_cstride, x_cstride, out_cstride;
  int n_chain;
  stp3_block_chain chain[3];
  int has_res_proj;           /* 1: residual = 1x1 projection of x (chain `res`, 64 outputs); 0: residual = x itself */
  stp3_block_chain res;
  int piece_col[16];
} stp3_block_desc;
size_t stp3_block_fused_scratch_bytes(int n_img);
int stp3_block_fused_fwd(const stp3_block_desc* desc, const void* mid_hi, const void* mid_lo, const void* x_hi,
                         const void* x_lo, const void* w, const float* hid_bias, const float* img_bias,
                         const float* res_bias, void* y_hi, void* y_lo, float* col_sums, void* scratch,
                         size_t scratch_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Memory-bound helpers of the dense path (all tensors channels-last bf16 hi/lo planes unless noted).
 * stp3_f32_to_hilo, stp3_hilo_to_f32 and stp3_spatial_sum take n_img <= 65535.
 */
/* fp32 (n_img,C,H,W) [channels_last=0, the reference's NCHW] or (n_img,H,W,C) [1] -> hi/lo (n_img,H,W,cp), padding 0.
 * Used where a foreign fp32 tensor enters a drop-in module (e.g. TemporalModel.forward, temporal_model.py:50). */
int stp3_f32_to_hilo(const float* x, int channels_last, int n_img, int C, int H, int W, int cp, void* hi, void* lo,
                     void* stream);
/* The one-plane counterpart: fp32 -> ONE plane (n_img,H,W,cp) of kind `operand` (STP3_OPERAND_BF16 or _F16), rounded
 * to nearest even (overflow to +-inf, NaN passes through), padding channels 0.  Same layouts and limits. */
int stp3_f32_to_plane(const float* x, int channels_last, int n_img, int C, int H, int W, int cp, int operand, void* out,
                      void* stream);
/* hi/lo (n_img,H,W,cstride) channels [c_off, c_off+C) -> fp32 (n_img,C,H,W): module outputs in the reference layout */
int stp3_hilo_to_f32(const void* hi, const void* lo, int n_img, int H, int W, int cstride, int c_off, int C, float* out,
                     void* stream);
/* sums[img][c] = sum over the H*W pixels (fp32, (n_img, cstride)); cstride <= 1024 */
int stp3_spatial_sum(const void* hi, const void* lo, int n_img, int HW, int cstride, float* sums, void* stream);
/* stp3_spatial_sum in a fixed order (the deterministic mode): per image and channel, fp64 partial sums of hi + lo over
 * fixed pixel ranges, added in range order and rounded once to fp32 -- the two passes of stp3_image_channel_sums.
 * The result depends on the input values and shape only.  Same arguments and limits (n_img <= 65535, cstride <= 1024);
 * scratch: stp3_spatial_sum_det_scratch_bytes(n_img, HW, cstride) bytes of device memory (no invariant). */
size_t stp3_spatial_sum_det_scratch_bytes(int n_img, int HW, int cstride);
int stp3_spatial_sum_det(const void* hi, const void* lo, int n_img, int HW, int cstride, float* sums, void* scratch,
                         size_t scratch_bytes, void* stream);
/* Spatially constant branches folded to a per-image bias of the consuming 1x1 convolution:
 *   m[c] = sums[c] * inv_hw for the C - n_const spatial channels, const_vals[img][c - (C - n_const)] for the trailing
 *       n_const spatially constant ones (their mean is the value); temporal != 0: averaged with the previous frame of
 *       the same sample when it exists -- AvgPool3d((2,H,W), padding (1,0,0), count_include_pad=False), temporal.py:397-415
 *   v = relu(W1 m + b1)  (R);   out[img][co] = (accumulate ? out[img][co] : bias ? bias[co] : 0) + sum_r W2[co][r] v[r]
 * C + R <= 12288 (m and v live in 48 KiB of shared memory).
 * Replaces PyramidSpatioTemporalPooling (temporal.py:375-423) and ASPPPooling (convolutions.py:227-239). */
int stp3_pool_bias(const float* sums, int sums_stride, int n_img, int T, int C, float inv_hw, int temporal,
                   const float* const_vals, int n_const, const float* W1, const float* b1, int R, const float* W2, int CO,
                   const float* bias, float* out, int co_stride, int accumulate, void* stream);
/* y[n][co] = (accumulate ? y[n][co] : bias ? bias[co] : 0) + sum_ci W[co][ci] x[n][ci]: the 6 broadcast ego-motion
 * channels of stp3.py:145-152 as a per-image bias */
int stp3_small_linear(const float* x, const float* W, int n, int ci, int co, const float* bias, float* y, int co_stride,
                      int accumulate, void* stream);
/* y[..., y_coff:y_coff+C] = bilinear_x2(x[..., :C]) (+ skip[..., s_coff:s_coff+C] when skip is given); x is
 * (n_img,h,w,.), skip and y are (n_img,2h,2w,.).  UpsamplingAdd tail (convolutions.py:204-215) and the upsample +
 * concat of UpsamplingConcat (convolutions.py:183-201).  16-byte vectors: every plane 16-byte aligned, C, the strides
 * and the offsets multiples of 8. */
int stp3_upsample2x_add(const void* x_hi, const void* x_lo, int n_img, int h, int w, int x_cstride, const void* s_hi,
                        const void* s_lo, int s_cstride, int s_coff, void* y_hi, void* y_lo, int y_cstride, int y_coff,
                        int C, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Train mode of the BEV decoder, the DeepLab head and the TemporalBlocks (stp3/models/decoder.py,
 * stp3/layers/convolutions.py:227-280, stp3/layers/temporal.py:252-489 in train(): BatchNorm with batch statistics,
 * dropout, autograd).
 * Tensors are fp32 channels-last (n_pix, cstride) with the channels at [0, C) of each row unless noted; every
 * reduction is deterministic (per-block partials in `scratch`, summed in a fixed order, no float atomics), so two calls
 * on the same inputs return bitwise-identical results.  The input gradient of a convolution is stp3_conv_fwd itself
 * (transposed weights, mirrored taps; stride 2 as four phase convolutions joined by stp3_phase_interleave).
 *
 * Weight gradient of a (kh x kw, stride, zero padding pad, dilation d >= 1) convolution, reference layout
 * (cout, cin, kh, kw):
 *   dw[co][ci][ky][kx] = sum over the n_img*Ho*Wo output pixels p of g[p][co] * x[p*stride + (ky*d-pad, kx*d-pad)][ci]
 *   x (n_img, H, W, x_cstride), g (n_img, Ho, Wo, g_cstride); scratch: stp3_conv_wgrad_scratch_bytes() bytes.
 *   A tap whose shifted window lies in the zero padding for every output pixel gets exact zeros (its pixels are not
 *   read).  The input gradient of a dilated convolution is stp3_conv_fwd with the mirrored taps e = pad - k*d. */
size_t stp3_conv_wgrad_scratch_bytes(int n_img, int Ho, int Wo, int cout, int cin, int kh, int kw, int dilation);
int stp3_conv_wgrad(const float* x, int n_img, int H, int W, int x_cstride, int cin, const float* g, int Ho, int Wo,
                    int g_cstride, int cout, int kh, int kw, int stride, int pad, int dilation, void* scratch,
                    size_t scratch_bytes, float* dw, void* stream);
/* Weight gradient of a causal (kt, kh, kw) 3-D convolution (stride 1, 'same' spatial padding (kh-1)/2, kh == kw odd,
 * time padded on the left by kt - 1: the TemporalBlock's CausalConv3d, temporal.py:252-269), reference layout
 * (cout, cin, kt, kh, kw):
 *   dw[co][ci][it][ky][kx] = sum over b, t and pixels of g[b][t][p][co] * x[b][t + it - (kt-1)][p + (ky, kx) - pad][ci]
 *   x (B, T, H, W, x_cstride), g (B, T, H, W, g_cstride); frames and pixels outside the tensor are zeros.  A time tap
 *   that reads padding for every output frame (kt - 1 - it >= T) stores exact zeros without reading pixels.
 *   scratch: stp3_conv3d_wgrad_scratch_bytes() bytes.  The same GEMM, split and ordered reduction as stp3_conv_wgrad
 *   (deterministic).  The input gradient is stp3_conv_fwd with the mirrored taps (kt-1-it, pad-ky, pad-kx): their time
 *   offsets are >= 0, and frames at or past T read as zero. */
size_t stp3_conv3d_wgrad_scratch_bytes(int B, int T, int H, int W, int cout, int cin, int kt, int kh, int kw);
int stp3_conv3d_wgrad(const float* x, int B, int T, int H, int W, int x_cstride, int cin, const float* g, int g_cstride,
                      int cout, int kt, int kh, int kw, void* scratch, size_t scratch_bytes, float* dw, void* stream);
/* One-product weight gradients: stp3_conv_wgrad / stp3_conv3d_wgrad on ONE 16-bit plane per operand (operand BF16 or
 * F16; x and g hold values of that kind, e.g. the planes the forward convolution and the input gradient read), one MMA
 * per 16-pixel k-slice instead of three.  Same arguments, layouts, argument checks and scratch queries
 * (stp3_conv_wgrad_scratch_bytes / stp3_conv3d_wgrad_scratch_bytes); the same K split, per-stage fp32 add into the
 * accumulator and ordered reduction, so two calls give bitwise-identical dw. */
int stp3_conv_wgrad_plane(int operand, const void* x, int n_img, int H, int W, int x_cstride, int cin, const void* g,
                          int Ho, int Wo, int g_cstride, int cout, int kh, int kw, int stride, int pad, int dilation,
                          void* scratch, size_t scratch_bytes, float* dw, void* stream);
int stp3_conv3d_wgrad_plane(int operand, const void* x, int B, int T, int H, int W, int x_cstride, int cin,
                            const void* g, int g_cstride, int cout, int kt, int kh, int kw, void* scratch,
                            size_t scratch_bytes, float* dw, void* stream);
/* BatchNorm batch statistics over n_pix rows (two passes: mean, then the centred sum of squares; fp64 partials):
 * mean[C], var[C] (biased; may be NULL), invstd = 1/sqrt(var + eps); when running_mean/var are given they are updated
 * like nn.BatchNorm2d: r = (1 - momentum) r + momentum b, with the unbiased variance var * n/(n-1).
 * scratch: stp3_bn_scratch_bytes(n_pix, C) bytes (also what stp3_bn_bwd_reduce needs). */
size_t stp3_bn_scratch_bytes(long long n_pix, int C);
int stp3_bn_stats(const float* x, long long n_pix, int C, int x_cstride, float eps, float momentum, float* running_mean,
                  float* running_var, float* mean, float* var, float* invstd, void* scratch, size_t scratch_bytes,
                  void* stream);
/* y = relu?((x - mean) * invstd * gamma + beta (+ res)) -> fp32 y (may be NULL) and/or bf16 hi/lo planes (n_pix,
 * hl_cstride) for the next stp3_conv_fwd (channels [C, hl_cstride) written as zeros).  Any C and fp32 row strides (8
 * channels per thread when C % 8 == 0 and every fp32 row is 16-byte aligned, else one element per thread: the same
 * values); the bf16 planes need hl_cstride % 8 == 0 and 16-byte alignment.
 * Dropout (0 <= dropout_p < 1; 0 = none, bit for bit): y is then multiplied by m / (1 - p), where the keep bit m of
 * element (pixel, c) depends only on (seed, offset + pixel * C + c): word e % 4 of Philox-4x32-10 with key seed and
 * counter (e / 4, 0) (64-bit values as (low, high) words), read as (word >> 8) / 2^24, keeps when it is >= p.  So a
 * tensor split across launches (offset = the elements before each part) gets the same mask as one launch.  Both y and
 * the bf16 planes carry the dropped values; a kept, positive element is exactly one with y > 0. */
int stp3_bn_apply(const float* x, long long n_pix, int C, int x_cstride, const float* mean, const float* invstd,
                  const float* gamma, const float* beta, const float* res, int res_cstride, int relu, float dropout_p,
                  unsigned long long seed, unsigned long long offset, float* y, int y_cstride, void* y_hi, void* y_lo,
                  int hl_cstride, void* stream);
/* stp3_bn_apply emitting ONE plane of kind `operand` (STP3_OPERAND_BF16 or _F16) instead of the hi/lo pair: y_plane
 * (n_pix, plane_cstride) receives the fp32 result y rounded to nearest even (overflow to +-inf, NaN passes through),
 * channels [C, plane_cstride) as zeros.  Same values of y, same dropout bits, same argument rules (y_plane follows the
 * rules of y_hi). */
int stp3_bn_apply_plane(const float* x, long long n_pix, int C, int x_cstride, const float* mean, const float* invstd,
                        const float* gamma, const float* beta, const float* res, int res_cstride, int relu,
                        float dropout_p, unsigned long long seed, unsigned long long offset, float* y, int y_cstride,
                        void* y_plane, int plane_cstride, int operand, void* stream);
/* sum_g[c] = sum_p g'[p][c] (= dbeta, or a conv bias gradient when x is NULL) and sum_gxhat[c] = sum_p g' xhat (= dgamma),
 * g' = g where y > 0 (the ReLU mask of the BN's activated output y; y NULL = no mask), xhat = (x - mean) * invstd. */
int stp3_bn_bwd_reduce(const float* g, int g_cstride, const float* y, int y_cstride, const float* x, int x_cstride,
                       const float* mean, const float* invstd, long long n_pix, int C, float* sum_g, float* sum_gxhat,
                       void* scratch, size_t scratch_bytes, void* stream);
/* sums[img][c] = sum over the hw rows of image img of x[img * hw + p][c], x (n_img * hw, x_cstride) fp32: per-image
 * channel sums in a fixed order (fp64 partials in scratch), bitwise repeatable -- the global-pool branch of the DeepLab
 * head and its backward.  sums (n_img, C); scratch: stp3_image_channel_sums_scratch_bytes() bytes. */
size_t stp3_image_channel_sums_scratch_bytes(int n_img, long long hw, int C);
int stp3_image_channel_sums(const float* x, int n_img, long long hw, int C, int x_cstride, float* sums, void* scratch,
                            size_t scratch_bytes, void* stream);
/* dx = gamma * invstd * (g' - sum_g/n - xhat * sum_gxhat/n); g_masked (optional) receives g' (the gradient of a residual
 * that was added before the ReLU).  Any C and row strides (vector path under the conditions of stp3_bn_apply). */
int stp3_bn_bwd_apply(const float* g, int g_cstride, const float* y, int y_cstride, const float* x, int x_cstride,
                      const float* mean, const float* invstd, const float* gamma, const float* sum_g,
                      const float* sum_gxhat, long long n_pix, int C, float* dx, int dx_cstride, float* g_masked,
                      int gm_cstride, void* stream);
/* SyncBatchNorm (statistics over every rank of a process group; the caller all-gathers the records between the local
 * and the merge calls).  A moments record is (4, C) fp64, rows n, S = sum x, Q = sum (x - m)^2, m = the fp32-rounded
 * local mean: stp3_bn_local_moments writes this rank's into out (e.g. its row of the gather buffer), with the two fixed
 * order passes of stp3_bn_stats; scratch: stp3_bn_scratch_bytes(n_pix, C).
 * stp3_bn_merge_finalize merges `world` records (world, 4, C) in rank order in fp64: N = sum n, mean = sum S / N,
 * M2 = sum_r Q_r - 2 (mean - m_r)(S_r - n_r m_r) + n_r (mean - m_r)^2, var = M2 / N (biased), invstd, and the running
 * statistics with the unbiased M2 / (N - 1), as stp3_bn_stats.  Every rank gets the same bits; world = 1 gives
 * stp3_bn_stats' bits. */
int stp3_bn_local_moments(const float* x, long long n_pix, int C, int x_cstride, double* out, void* scratch,
                          size_t scratch_bytes, void* stream);
int stp3_bn_merge_finalize(const double* records, int world, int C, float eps, float momentum, float* running_mean,
                           float* running_var, float* mean, float* var, float* invstd, void* stream);
/* Backward of a SyncBatchNorm: stp3_bn_bwd_local_sums writes this rank's (2, C) fp64 record (sum g', sum g' xhat) over
 * its n_pix rows (the arguments of stp3_bn_bwd_reduce); stp3_bn_bwd_merge_sums adds `world` records (world, 2, C) in
 * rank order into fp32 sum_g / sum_gxhat (world = 1: stp3_bn_bwd_reduce's bits); stp3_bn_bwd_apply_global is
 * stp3_bn_bwd_apply over this rank's n_pix rows with the group's merged sums and row count n_total:
 * dx = gamma * invstd * (g' - sum_g/n_total - xhat * sum_gxhat/n_total). */
int stp3_bn_bwd_local_sums(const float* g, int g_cstride, const float* y, int y_cstride, const float* x, int x_cstride,
                           const float* mean, const float* invstd, long long n_pix, int C, double* out, void* scratch,
                           size_t scratch_bytes, void* stream);
int stp3_bn_bwd_merge_sums(const double* records, int world, int C, float* sum_g, float* sum_gxhat, void* stream);
int stp3_bn_bwd_apply_global(const float* g, int g_cstride, const float* y, int y_cstride, const float* x,
                             int x_cstride, const float* mean, const float* invstd, const float* gamma,
                             const float* sum_g, const float* sum_gxhat, long long n_pix, long long n_total, int C,
                             float* dx, int dx_cstride, float* g_masked, int gm_cstride, void* stream);
/* bilinear x2 (align_corners=False, nn.Upsample of UpsamplingAdd) on fp32 (n_img, h, w, C) -> (n_img, 2h, 2w, C), and
 * its adjoint (a gather over the outputs each input feeds; no atomics) */
int stp3_upsample2x_f32(const float* x, int n_img, int h, int w, int C, float* y, void* stream);
int stp3_upsample2x_bwd(const float* gy, int n_img, int h, int w, int C, float* gx, void* stream);
/* The same pair on a channel window of a wider channels-last tensor (the concat tensor of UpsamplingConcat in train
 * mode, convolutions.py:183-201: the upsampled coarse map sits behind the fine map, and its gradient is read from there):
 *   forward: x dense (n_img, h, w, C) -> channels [y_coff, y_coff + C) of y (n_img, 2h, 2w, y_cstride); the other
 *            channels of y are not touched
 *   adjoint: channels [gy_coff, gy_coff + C) of gy (n_img, 2h, 2w, gy_cstride) -> gx dense (n_img, h, w, C)
 * 16-byte accesses when C, the row stride and the offset are multiples of 4 and both pointers are 16-byte aligned, one
 * float per thread otherwise: the same values.  With the stride C and offset 0 these are the two functions above. */
int stp3_upsample2x_window_f32(const float* x, int n_img, int h, int w, int C, float* y, int y_cstride, int y_coff,
                               void* stream);
int stp3_upsample2x_window_bwd(const float* gy, int gy_cstride, int gy_coff, int n_img, int h, int w, int C, float* gx,
                               void* stream);
/* out (n_img, H, W, C)[y][x] = p_{y%2 x%2}[y/2][x/2], phase p_ab of size (n_img, (H-a+1)/2, (W-b+1)/2, C) or NULL = 0:
 * the four phases of a stride-2 convolution's input gradient */
int stp3_phase_interleave(const float* p00, const float* p01, const float* p10, const float* p11, int n_img, int H, int W,
                          int C, float* out, void* stream);
/* dz = g * s * (1 - s), s = sigmoid(z) the forward output (instance_center head, decoder.py:70) */
int stp3_sigmoid_bwd(const float* g, const float* s, long long n, float* dz, void* stream);
/* The pyramid-pooling branch of a TemporalBlock in time (AvgPool3d((2, H, W)), time padding 1,
 * count_include_pad=False; temporal.py:375-423) on per-frame means m (B, T, C) fp32:
 *   adjoint == 0: the T + 1 pooled frames out (B, T + 1, C): out[b][0] = m[b][0], out[b][t] = (m[b][t-1] + m[b][t]) / 2
 *   for 1 <= t < T, out[b][T] = m[b][T-1].  The reference drops frame T only after the branch's BatchNorm, so its
 *   batch statistics cover B * (T + 1) values.
 *   adjoint != 0 (its transpose): m is a gradient (B, T + 1, C), out (B, T, C): out[b][t] = c_t m[b][t] + m[b][t+1] / 2
 *   for t + 1 < T, c_t m[b][t] + m[b][T] for t = T - 1; c_0 = 1, c_t = 1/2 for t >= 1.  out must not alias m. */
int stp3_temporal_pair_mean(const float* m, int B, int T, int C, int adjoint, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * EfficientNet trunk (efficientnet-pytorch 0.7.0, truncated like stp3/models/encoder.py:39-55).  The 1x1 expand and
 * projection convolutions of an MBConv block are stp3_conv_fwd calls (swish, per-image weights); these are the rest.
 * Static "same" padding: pad_t / pad_l are the top / left pads computed for the model's nominal image size; inputs
 * outside the image read as zero, which is the bottom / right pad.  BatchNorm (eps 1e-3) is folded by the caller.
 *
 * Stem: fp32 NCHW images (n_img, 3, H, W) -> 3x3 stride-2 conv (w [cout][3][3][3], bias [cout]) + swish -> hi/lo planes
 * (n_img, Ho, Wo, out_cstride); channels [cout, out_cstride) are written as zeros.  cout <= 64, out_cstride a multiple
 * of 64, y_hi / y_lo 16-byte aligned, n_img * Ho * Wo * out_cstride / 16 threads in at most 2^31 - 1 blocks of 256. */
int stp3_effnet_stem(const float* x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, const float* w,
                     const float* bias, int cout, int out_cstride, void* y_hi, void* y_lo, void* stream);
/* Depthwise k x k convolution (k 3 or 5, stride 1 or 2) + folded BN + swish on hi/lo planes, channels [0, C) of
 * x (n_img, H, W, in_cstride) -> y (n_img, Ho, Wo, out_cstride); other channels of y are not touched.  w [k*k][C] fp32,
 * bias [C].  sums (optional, (n_img, C) fp32): per-(image, channel) sums of the activated output -- the squeeze-excite
 * means -- through stp3_dw_sums_scratch_bytes(desc) bytes of scratch and a fixed-order reduction (bitwise repeatable). */
typedef struct stp3_dw_desc {
  int n_img, H, W, Ho, Wo;
  int k, stride, pad_t, pad_l;
  int C;                 /* multiple of 8; padding channels with zero weights and bias come out zero */
  int in_cstride, out_cstride;   /* multiples of 64 */
} stp3_dw_desc;
size_t stp3_dw_sums_scratch_bytes(const stp3_dw_desc* desc);
int stp3_dw_fwd(const stp3_dw_desc* desc, const void* x_hi, const void* x_lo, const float* w, const float* bias,
                void* y_hi, void* y_lo, float* sums, void* scratch, size_t scratch_bytes, void* stream);
/* Squeeze-excite gate of every image, gate = sigmoid(w_e . swish(w_r . (sums * inv_hw) + b_r) + b_e) (w_r [R][C],
 * w_e [C][R]), folded into per-image projection weights w_img = W_proj . diag(gate) (w_proj [cout][C] fp32, BN folded)
 * in the packed hi/lo layout of stp3_conv_fwd: per image stp3_se_proj_weight_elems(C, cout) bf16 elements holding column
 * chunks of 128 output channels (the last one 64 or 128 rows wide, zero padded), chunk j at the offset of the chunks
 * before it, each [C/64 rounded up][2][bn_j][64].  gate (n_img, C) fp32 receives the gate (computed once per image by a
 * first kernel; a second one scales the weights). */
long long stp3_se_proj_weight_elems(int cin, int cout);
int stp3_se_gate(const float* sums, int sums_stride, int n_img, int C, float inv_hw, const float* w_r, const float* b_r,
                 int R, const float* w_e, const float* b_e, const float* w_proj, int cout, float* gate, void* w_img,
                 void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * EfficientNet trunk, train mode (EfficientNetTrunk(trainable=True).train()).  fp32 channels-last tensors with C
 * channels per pixel row unless a stride says otherwise; the static pads are the eval kernels' (top / left from the
 * nominal image size, zero past the bottom / right edge).  Reductions write per-block fp64 partials into caller scratch
 * and add them in a fixed order: no atomics, bitwise repeatable.  1x1 convolutions, their gradients, the batch
 * statistics and the BatchNorm backward are the decoder's train-mode entry points above.
 *
 * stp3_effnet_stem_raw: y (n_img, Ho, Wo, cout) = 3x3 stride-2 conv of the NCHW images x (n_img, 3, H, W) with
 * w [cout][3][3][3], no bias, no activation.  cout <= 64.
 * stp3_effnet_stem_wgrad: dw [cout][3][3][3] = sum over images and output pixels of g (n_img, Ho, Wo, cout) times the
 * input tap the forward read (zero outside the image), through stp3_effnet_stem_wgrad_scratch_bytes() of scratch. */
int stp3_effnet_stem_raw(const float* x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, const float* w,
                         int cout, float* y, void* stream);
size_t stp3_effnet_stem_wgrad_scratch_bytes(int n_img, int Ho, int Wo, int cout);
int stp3_effnet_stem_wgrad(const float* x, int n_img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, const float* g,
                           int cout, float* dw, void* scratch, size_t scratch_bytes, void* stream);
/* Depthwise k x k (3 / 5), stride 1 / 2, on fp32 tensors described by stp3_dw_desc with in_cstride / out_cstride in
 * fp32 elements (>= C, any C):
 * stp3_dw_fwd_raw: y (n_img, Ho, Wo, .) = the convolution of x (n_img, H, W, .) with w [k*k][C], no bias, no activation.
 * stp3_dw_dgrad: dx (n_img, H, W, .) = its exact adjoint applied to g (n_img, Ho, Wo, .): every input pixel gets the taps
 * that read it; pixels no output read (past the bottom / right edge) get zero.
 * stp3_dw_wgrad: dw [k*k][C] = sum over images and output pixels of g times the input tap, through
 * stp3_dw_wgrad_scratch_bytes(desc) of scratch. */
int stp3_dw_fwd_raw(const stp3_dw_desc* desc, const float* x, const float* w, float* y, void* stream);
int stp3_dw_dgrad(const stp3_dw_desc* desc, const float* g, const float* w, float* dx, void* stream);
size_t stp3_dw_wgrad_scratch_bytes(const stp3_dw_desc* desc);
int stp3_dw_wgrad(const stp3_dw_desc* desc, const float* x, const float* g, float* dw, void* scratch,
                  size_t scratch_bytes, void* stream);
/* stp3_trunk_bn_act: y = act(z) * mul[img][c] * scale[img] + res over x (n_pix, C), img = pixel / img_pix, with
 * z = (x - mean) * invstd * gamma + beta (batch statistics of stp3_bn_stats; z = x when mean is NULL) and act swish
 * (swish != 0) or the identity.  mul (n_img, C), scale (n_img), res (n_pix, C) are optional.  Writes y (n_pix, C) fp32
 * and / or the hi/lo planes (n_pix, hl_cstride) of the next convolution, columns [C, hl_cstride) as zeros.
 * The MBConv uses: _bn0 / _bn1 / stem + swish; the squeeze-excite gate (no statistics, mul = gate); _bn2 with the
 * drop-connect scale and the identity skip.
 * stp3_trunk_bn_act_bwd: out = (g * mul[img][c] + add[img][c]) * act'(z) * scale[img], z recomputed from x; the
 * dL/dz stp3_bn_bwd_reduce / stp3_bn_bwd_apply (or their SyncBatchNorm forms) then take with no ReLU mask.  out must
 * not alias g. */
int stp3_trunk_bn_act(const float* x, long long n_pix, int C, long long img_pix, const float* mean, const float* invstd,
                      const float* gamma, const float* beta, int swish, const float* mul, const float* scale,
                      const float* res, float* y, void* y_hi, void* y_lo, int hl_cstride, void* stream);
int stp3_trunk_bn_act_bwd(const float* g, const float* x, long long n_pix, int C, long long img_pix, const float* mean,
                          const float* invstd, const float* gamma, const float* beta, int swish, const float* mul,
                          const float* add, const float* scale, float* out, void* stream);
/* stp3_image_channel_dot: out (n_img, C) = per image and channel, the sum over its hw pixels of a * b (a, b
 * (n_img, hw, C)): the squeeze-excite gate gradient sum_p y * (W_proj^T dz). */
size_t stp3_image_channel_dot_scratch_bytes(int n_img, long long hw, int C);
int stp3_image_channel_dot(const float* a, const float* b, int n_img, long long hw, int C, float* out, void* scratch,
                           size_t scratch_bytes, void* stream);
/* stp3_se_bwd: one CTA per image, from dgate (n_img, C), the forward's gate (n_img, C) and spatial sums (n_img, C):
 * m = sums * inv_hw, r = w_r m + b_r (w_r [R][C]), de = dgate * gate * (1 - gate) (n_img, C), sr = swish(r) (n_img, R),
 * dr = (w_e^T de) * swish'(r) (n_img, R) (w_e [C][R]), dmean = (w_r^T dr) * inv_hw (n_img, C): the gradient of the
 * squeeze-excite mean spread over each pixel.  The weight gradients are dW_e = de^T sr, dW_r = dr^T m and the bias
 * gradients the column sums of de and dr. */
int stp3_se_bwd(const float* dgate, const float* gate, const float* sums, int n_img, int C, float inv_hw,
                const float* w_r, const float* b_r, int R, const float* w_e, float* de, float* sr, float* dr,
                float* dmean, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Discount recurrence of the frame-sharded lift-splat (stp3_lift_splat_fwd with f_count > 0), after the all-gather */
int stp3_bev_discount(const float* raw /*(B,S,nx,ny,C) fp32*/, int B, int S, int nx, int ny, int C, float discount,
                      void* out_hi, void* out_lo /*(B,S,nx,ny,C) bf16 each*/, void* stream);


/* ---------------------------------------------------------------------------------------------------------
 * Prediction stage (eval mode, N_FUTURE_FRAMES > 0): the per-pixel kernels between the stage's convolutions
 *   DistributionModule / Bottleneck(downsample)   stp3/models/distributions.py, stp3/layers/convolutions.py:65-170
 *   Dual_GRU, SpatialGRU                          stp3/layers/temporal.py:11-160
 *   LayerNorm, Block (ConvNeXt), Bottleblock      stp3/layers/convolutions.py:283-380
 *
 * stp3_hl_slot: a channel slot of a channels-last bf16 hi/lo activation (B, t_total, H, W, cstride) -- channels
 * [coff, coff + C) of frames [t0, t0 + T) of every sample, where a call processes B samples of T frames.  cstride and
 * coff are multiples of 8 and both planes 16-byte aligned.  Each call reads and writes only its slots; channels outside
 * them are untouched.  Every result is a fixed-order fp32 function of its inputs (no atomics): repeated launches are
 * bitwise equal. */
typedef struct {
  void* hi;
  void* lo;
  int cstride, coff;
  int t_total, t0;
} stp3_hl_slot;

/* out = (1 - sigmoid(r)) * h: the reset-gated state of a conv-GRU proposal (r is the raw reset-gate convolution) */
int stp3_gru_gates(const stp3_hl_slot* r, const stp3_hl_slot* h, const stp3_hl_slot* out, int B, int T, long long HW,
                   int C, void* stream);
/* out [and out2 when not NULL] = (1 - s) * h + s * h_tilde, s = sigmoid(u) (u the raw update-gate convolution); out
 * may be the slot of h itself */
int stp3_gru_update(const stp3_hl_slot* u, const stp3_hl_slot* h, const stp3_hl_slot* h_tilde, const stp3_hl_slot* out,
                    const stp3_hl_slot* out2, int B, int T, long long HW, int C, void* stream);
/* out = act(LN(x)) + act_y(y), per pixel over its C <= 256 channels: LN with gamma / beta (C) fp32 and eps, biased
 * variance (skipped when gamma and beta are NULL); act = exact GELU when gelu != 0; y optional (NULL: nothing added),
 * act_y = exact GELU when gelu_y != 0.  out may be the slot of x. */
int stp3_channel_norm_act(const stp3_hl_slot* x, const float* gamma, const float* beta, float eps, int gelu,
                          const stp3_hl_slot* y, int gelu_y, const stp3_hl_slot* out, int B, int T, long long HW, int C,
                          void* stream);
/* out = LN(depthwise k x k convolution of x (zero padding k/2, stride 1) + bias): w (k*k, C) fp32 tap-major, 16-byte
 * aligned, bias / gamma / beta (C) fp32, C <= 256; out's planes must not overlap x's (not even in other channels or
 * frames of the same buffer: the call refuses any overlap of the two slots' address spans) */
int stp3_dw_ln(const stp3_hl_slot* x, const float* w, const float* bias, int k, const float* gamma, const float* beta,
               float eps, const stp3_hl_slot* out, int B, int T, int H, int W, int C, void* stream);
/* The trusting gate's tail (temporal.py:110-115): z = w t (w (2, C) fp32, C <= 256), p = softmax(z),
 * mix = s2 * p0 + s1 * p1, written to each of the n_dst (1..4) slots of dst (a host array) */
int stp3_trust_mix(const stp3_hl_slot* t, const float* w, const stp3_hl_slot* s1, const stp3_hl_slot* s2,
                   const stp3_hl_slot* dst, int n_dst, int B, int T, long long HW, int C, void* stream);
/* out (ceil(H/2), ceil(W/2)) = MaxPool2d(2, 2) of x after an odd H / W was zero-padded by one row / column at the
 * bottom / right (convolutions.py:160-164: the padded zeros take part in the max); the winning hi / lo bits are
 * stored unchanged */
int stp3_maxpool2_pad(const stp3_hl_slot* x, const stp3_hl_slot* out, int B, int T, int H, int W, int C, void* stream);
/* dst = src (C channels of every pixel, both planes bit for bit) */
int stp3_hl_copy(const stp3_hl_slot* src, const stp3_hl_slot* dst, int B, int T, long long HW, int C, void* stream);
/* dst[img, pixel, c] = vec[img * vstride + c] (img = b * T + t): a per-image vector broadcast over H x W */
int stp3_hl_broadcast(const float* vec, int vstride, const stp3_hl_slot* dst, int B, int T, long long HW, int C,
                      void* stream);

/* ============================================================================================================
 * Eval-mode planning (stp3/models/planning_model.py, stp3/cost.py): the cost of every sampled trajectory at every
 * future frame, the choice of the cheapest one within a command window, and the GRU refinement of that choice.
 *
 * stp3_plan_desc describes the call.  The footprints are the integer (row, col) cells of the ego rectangle that
 * BaseCost.get_origin_points rasterises (cost.py:68-81), without and with the safety margin lambda; both are full
 * rectangles [r0, r1] x [c0, c1] of absolute BEV cells (rows and columns >= 0).
 *
 * Layouts (fp32 unless noted; B samples, N candidates, T future frames, H x W BEV cells):
 *   lane, drivable  (B, n_hd, H, W): the lane-divider and drivable-area channels of the hd map -- two logits per
 *                   element (n_hd 2: softmax, channel 1) or the raw map (n_hd 1)
 *   drv_map         (B, H, W): drivable probability, 0 where it is < 0.5 (the raw channel when n_hd is 1)
 *   dang_map        (B, H, W) uint8: 1 where drv_map is 0 (Rule's dangerous area)
 *   lane_cost       (B, H, W): LR_divider's cost at every cell, lrdivider * (L - d)^2 where the distance d to the
 *                   nearest lane cell is <= L = lane_dist, else 0
 *   trajs           (B, N, T, traj_c): x, y (and a third component the cost ignores) of every candidate
 *   occupancy       (B, T, H, W) uint8 0 / 1: the predicted vehicle-or-pedestrian occupancy
 *   cost_volume     (B, T, H, W)
 *   target_points   (B, 2)
 *   cost_fc         (B, N) and cost_fo (B, N, T): Cost_Function.forward's two results
 *   windows         (B, 2) int32 device array of (first candidate, count) per sample; windows_host the same values
 *                   on the host (checked before the launch)
 *   h0              (B, G): the reduced front-camera features, the GRU's initial state
 *   w_ih (3G, 6), b_ih (3G), w_hh_t (G, 3G) = GRUCell.weight_hh transposed, b_hh (3G), gate order (r, z, n);
 *   w1_t (G, G) = decoder[0].weight transposed, b1 (G), w2 (2, G), b2 (2)
 *   out_traj        (B, T, 3): the refined trajectory, third column 0
 *   selected        (B) int32: index into trajs of the candidate chosen in the sample's window (lowest on ties)
 * No atomics, and nothing is read back to the host: repeated calls are bitwise equal. */
typedef struct stp3_plan_desc {
  int B, N, T;                  /* N a multiple of 3; 1 <= T <= 16 */
  int H, W;                     /* BEV rows x columns (bev_dimension[0], [1]); H == W */
  float dx[2], bx[2];           /* BaseCost.dx, BaseCost.bx (fp32) */
  int fp0[4];                   /* footprint at lambda 0: first row, last row, first column, last column */
  int fp1[4];                   /* footprint at lambda: the same */
  float safety, headway, lrdivider, comfort, progress, volume;   /* COST_FUNCTION factors */
  float rule;                   /* Rule.factor (5) */
  float safety_w[2];            /* SafetyCost.w */
  float headway_dist;           /* HeadwayCost.L, metres added to y (10) */
  float lane_dist;              /* LR_divider.L, metres (1) */
  int n_hd;                     /* 1 or 2 channels per hd-map element */
  int traj_c;                   /* components per trajectory point: 2 or 3 */
  int G;                        /* GRU state size: a multiple of 32, at most 512 (stp3_plan_refine) */
} stp3_plan_desc;

/* One thread per (sample, cell): drv_map, dang_map and lane_cost */
int stp3_plan_maps(const stp3_plan_desc* desc, const float* lane, const float* drivable, float* drv_map,
                   uint8_t* dang_map, float* lane_cost, void* stream);
/* One warp per (sample, candidate, frame): cost_fc and cost_fo, every term clamped as Cost_Function.forward does */
int stp3_plan_cost(const stp3_plan_desc* desc, const float* trajs, const uint8_t* occupancy, const float* cost_volume,
                   const float* target_points, const float* drv_map, const uint8_t* dang_map, const float* lane_cost,
                   float* cost_fc, float* cost_fo, void* stream);
/* One CTA per sample: argmin of cost_fc + sum_t cost_fo over the window, then T GRUCell(6, G) steps with the
 * Linear(G, G) -> ReLU -> Linear(G, 2) decoder */
int stp3_plan_refine(const stp3_plan_desc* desc, const int32_t* windows_host, const int32_t* windows,
                     const float* trajs, const float* cost_fc, const float* cost_fo, const float* h0,
                     const float* target_points, const float* w_ih, const float* b_ih, const float* w_hh_t,
                     const float* b_hh, const float* w1_t, const float* b1, const float* w2, const float* b2,
                     float* out_traj, int32_t* selected, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STP3_B200_H_ */

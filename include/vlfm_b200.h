/*
 * vlfm_b200 -- C-ABI of the VLFM perception -> value-map hot path, written for the NVIDIA H100 (sm_90a).
 *
 * The reference (bdaiinstitute/vlfm) is pure Python: the boundary it exposes is a
 * Python class surface (vlfm/mapping/*.py, vlfm/vlm/*.py).  This header is the
 * thin C-ABI those classes are re-hosted on (vlfm_b200/mapping, vlfm_b200/vlm load it
 * with ctypes).  Every entry point cites the reference function it replaces.
 *
 * Conventions
 *   - plain C types only; `d_` pointers are DEVICE pointers, `h_` pointers are HOST.
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*),
 *     never allocates device memory and never synchronises unless documented.
 *   - return value: 0 (VLFM_OK) or a VLFM_E_* code; vlfm_last_error() gives text.
 *   - batched: `batch` environments per call; env b uses grid slot
 *     d_slot[b] (or b when d_slot == NULL) of the [nslots, G, G(, C)] state tensors.
 *   - per-environment soft errors (camera off-grid, scatter out of range) are
 *     reported through `d_status[b]` bit flags (VLFM_ST_*), read by the host at its
 *     next synchronisation point and turned into the reference's exceptions.
 */
#ifndef VLFM_B200_H_
#define VLFM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VLFM_OK 0
#define VLFM_E_INVALID 1   /* bad argument */
#define VLFM_E_CUDA 2      /* CUDA runtime error, see vlfm_last_error() */
#define VLFM_E_UNSUPPORTED 3
#define VLFM_E_DRIVER 4    /* driver entry point (TMA descriptor encode) unavailable */

/* d_status bits */
#define VLFM_ST_CAMERA_OFF_GRID 1  /* img_utils.py:43 assert -> AssertionError */
#define VLFM_ST_SCATTER_OOB 2      /* numpy IndexError in obstacle_map.py:101 */
#define VLFM_ST_FRONTIER_OVERFLOW 4

/* fusion modes (vlfm/mapping/value_map.py:357-429) */
#define VLFM_FUSE_WEIGHTED 0      /* use_max_confidence=False, fusion_type="default" */
#define VLFM_FUSE_MAX_CONFIDENCE 1 /* use_max_confidence=True */
#define VLFM_FUSE_REPLACE 2        /* fusion_type="replace" */
#define VLFM_FUSE_EQUAL 4          /* OR-ed flag: fusion_type="equal_weighting" */

const char* vlfm_last_error(void);
int vlfm_version(void);
/* number of kernels this library has launched since load (bench `gpu_launches`). */
unsigned long long vlfm_launch_count(void);

/* ------------------------------------------------------------------ value map ---- */
/* Replaces ValueMap.update_map (vlfm/mapping/value_map.py:100-128), i.e.
 * _process_local_data (:221-286), _localize_new_data (:288-319), rotate_image
 * (vlfm/utils/img_utils.py:9-28), place_img_in_img (:31-61), _fuse_new_data
 * (value_map.py:357-429).                                                          */
typedef struct VlfmValueParams {
  int32_t H, W;          /* depth image rows, cols                                   */
  int32_t G;             /* grid side (BaseMap.size, base_map.py:15)                 */
  int32_t C;             /* value channels                                           */
  int32_t R;             /* cone template side = 2*int(max_depth*ppm)+1 (:323)       */
  int32_t ppm;           /* pixels per metre                                         */
  float depth_scale;     /* (float)(max_depth - min_depth)     (value_map.py:234)    */
  float depth_offset;    /* (float)min_depth                                         */
  float decision_threshold; /* 0.35 (value_map.py:41)                                */
  int32_t fusion;        /* VLFM_FUSE_*                                              */
  int32_t rows_per_tile; /* fuse-kernel tiling; 0 = choose from batch               */
} VlfmValueParams;

/* bytes of scratch needed for `batch` environments. */
int vlfm_value_workspace_bytes(const VlfmValueParams* p, int batch, size_t* bytes);

/* d_conf   [nslots, G, G]    float32  (ValueMap._map)
 * d_value  [nslots, G, G, C] float32  (ValueMap._value_map)
 * d_depth  [batch, H, W]     float32 in [0,1]
 * d_tf     [batch, 16]       float64 row-major camera->episodic
 * d_values [batch, C]        float64
 * d_template [R, R]          float32 cone template (value_map.py:337-355; constant per
 *                            (fov, max_depth, ppm), built once by the host class)
 * d_tan    [W]               float64 tan(linspace(-fov/2, fov/2, W)) (value_map.py:237)
 * d_explored [nslots, G, G]  uint8 or NULL (value_map.py:369-375 masking of the new
 *                            observation; the full-grid part is vlfm_value_mask_unexplored)
 * d_workspace                vlfm_value_workspace_bytes(), must be zero-filled once
 * d_status [batch]           int32, OR-ed with VLFM_ST_* flags                        */
int vlfm_value_update(const VlfmValueParams* p, int batch, const int32_t* d_slot,
                      float* d_conf, float* d_value, const float* d_depth,
                      const double* d_tf, const double* d_values,
                      const float* d_template, const double* d_tan,
                      const uint8_t* d_explored, void* d_workspace, int32_t* d_status,
                      void* stream);

/* value_map.py:369-375: conf/value := 0 where explored == 0, over the whole grid. */
int vlfm_value_mask_unexplored(int G, int C, int batch, const int32_t* d_slot, float* d_conf,
                               float* d_value, const uint8_t* d_explored, void* stream);

/* Replaces ValueMap.sort_waypoints' inner pixel_value_within_radius
 * (value_map.py:163-176, img_utils.py:213-266): median of the non-zero cells of
 * channel c inside the radius-`radius` disc (d_disc: (2r+1)^2 uint8 mask as drawn by
 * cv2.circle) around (row,col) = d_points[i]; -1 when empty.
 * d_out [npoints, C] float64.                                                       */
int vlfm_value_disc_median(int G, int C, int slot, const float* d_value, const int32_t* d_points,
                           int npoints, int radius, const uint8_t* d_disc, double* d_out,
                           void* stream);
/* The same for the frontiers of MANY environments in one launch: d_points_srl [npoints,3] int32 = (slot, row, col),
 * d_value [nslots,G,G,C]; d_out [npoints,C].  (ITMPolicy._sort_frontiers_by_value, itm_policy.py:263-294, per env.) */
int vlfm_value_disc_median_batch(int G, int C, const float* d_value, const int32_t* d_points_srl, int npoints, int radius,
                                 const uint8_t* d_disc, double* d_out, void* stream);

/* --------------------------------------------------------------- obstacle map ---- */
/* Replaces ObstacleMap.update_map obstacle half (vlfm/mapping/obstacle_map.py:86-109):
 * hole fill (hole_area_thresh == -1 form), depth -> metres, get_point_cloud
 * (geometry_utils.py:216-236), transform_points (:205-213), filter_points_by_height
 * (obstacle_map.py:196-197), _xy_to_px (base_map.py:35-46), scatter, k x k dilation. */
typedef struct VlfmObstacleParams {
  int32_t H, W, G, ppm;
  float depth_scale;    /* (float)(max_depth - min_depth) */
  float depth_offset;   /* (float)min_depth               */
  float max_depth_f32;  /* (float)max_depth, mask = scaled < max_depth (:93)          */
  double fx, fy;
  double min_height, max_height;
  int32_t kernel;       /* odd dilation size (:43-46)                                 */
  int32_t full_grid;    /* 1: dilate whole grid (first update after reset); 0: ROI    */
  int32_t roi_half;     /* ROI half-size in cells around the camera cell              */
} VlfmObstacleParams;

/* d_obst [nslots,G,G] uint8 (ObstacleMap._map), d_nav [nslots,G,G] uint8
 * (ObstacleMap._navigable_map as 0/1).                                               */
/* d_hole_fill [batch,H,W] uint8 or NULL: output of vlfm_fill_small_holes (pixels whose depth becomes 1.0);
 * NULL selects the hole_area_thresh == -1 form (every zero depth becomes 1.0, obstacle_map.py:87-89). */
int vlfm_obstacle_update(const VlfmObstacleParams* p, int batch, const int32_t* d_slot,
                         uint8_t* d_obst, uint8_t* d_nav, const float* d_depth,
                         const double* d_tf, const uint8_t* d_hole_fill, int32_t* d_status, void* stream);
/* fill_small_holes (vlfm/utils/img_utils.py:361-390): zero-depth regions AND the islands they enclose whose
 * cv2.contourArea (RETR_TREE borders) is below area_thresh; d_filled [H,W] uint8 := 1 on the pixels set to 1.0. */
int vlfm_holes_workspace_bytes(int H, int W, size_t* bytes);
int vlfm_fill_small_holes(const float* d_depth, int H, int W, double area_thresh, uint8_t* d_filled, void* d_workspace,
                          int32_t* d_status, void* stream);

/* ---------------------------------------------------------------- dense (VLM) ---- */
/* fp16 x fp16 -> fp32-accumulate GEMM on Hopper tensor cores (wgmma), TMA-fed:
 *   out[M,N] = epilogue(A[M,K] @ W[N,K]^T + bias[N])
 * A, W row-major fp16 (K contiguous, K % 8 == 0).
 * epilogue: 0 = bias -> fp16 out; 1 = bias + GELU(erf) -> fp16 out;
 *           2 = bias + residual: resid_f32[M,N] += result (fp32 stream, in place)
 *           3 = bias -> fp32 out; 4 = bias + ReLU -> fp16 out (GroundingDINO FFNs)
 * These replace the nn.Linear calls inside lavis' Blip2 ITM forward
 * (reference call site vlfm/vlm/blip2itm.py:52).                                     */
#define VLFM_EPI_BIAS_F16 0
#define VLFM_EPI_BIAS_GELU_F16 1
#define VLFM_EPI_BIAS_RESID_F32 2
#define VLFM_EPI_BIAS_F32 3
#define VLFM_EPI_BIAS_RELU_F16 4
#define VLFM_EPI_PARTIAL_F32 5   /* internal to vlfm_gemm_f16_resid_ln: split-K partial sums stored side by side */
/* x[M,N] (fp32 residual stream) += A @ W^T + bias, then LayerNorm(x) -> d_out16 (fp16) and/or d_out32 (fp32, may
 * alias x for the post-LN Q-Former blocks).  BITWISE REPRODUCIBLE: when the tile plan splits K, the splits store their
 * partial sums in d_partials (no atomics) and the LayerNorm launch adds them to x in K order before normalising.  Below one
 * wave of 128 x 128 tiles the split is stream-K over one CTA per SM: (SMs + tiles - 1) slabs of 130 x 128 floats (66.5 KB);
 * a smaller d_partials lowers the CTA count, and below tiles + 1 CTAs the GEMM runs unsplit.  Above one wave the splits are
 * uniform (>= splits * M * N floats, splits <= 8); without d_partials (or when it is too small) they run unsplit: this
 * call never reduces with red.global.add (only vlfm_gemm_f16 with VLFM_EPI_BIAS_RESID_F32 does).  Stream-K results depend on
 * the SM count: bitwise reproducible across cards with the same count.
 * Replaces `x = x + proj(...)` followed by `layer_norm` in the BLIP-2 forward (blip2itm.py:52 through lavis).            */
int vlfm_gemm_f16_resid_ln(const void* d_A, const void* d_W, const float* d_bias, float* d_x, int M, int N, int K,
                           int lda, int ldw, int ldx, const float* d_gamma, const float* d_beta, void* d_out16, int ld16,
                           float* d_out32, int ld32, float eps, float* d_partials, size_t partial_bytes, void* stream);
/* the reduction + LayerNorm launch on its own: x += sum_s partials[s] (s ascending), out = LayerNorm(x) */
int vlfm_layernorm_reduce(float* d_x, const float* d_partials, int splits, long long split_stride, const float* d_gamma,
                          const float* d_beta, void* d_out16, float* d_out32, int rows, int D, int ldx, int ldo16, int ldo32,
                          float eps, void* stream);
int vlfm_gemm_f16(const void* d_A, const void* d_W, const float* d_bias, void* d_out, int M, int N,
                  int K, int lda, int ldw, int ldo, int epilogue, void* stream);
/* Epilogue flag of vlfm_gemm_f16 (OR it into the epilogue code): the caller allows the batch-1 ViT plan, whose summation order
 * differs from the plan for other row counts.  At 256 < M <= 258 the GEMM then runs one 256-row tile per column block and splits
 * K over a thread-block cluster, reduced in shared memory in rank order (bitwise reproducible, no atomics, residual epilogue
 * included).  Other M, weights below 8 Mi elements (there it measured slower), or VLFM_GEMM_CSPLIT=0 in the environment ignore
 * it; VLFM_GEMM_CSPLIT=2 takes it for any weight size.  vlfm_gemm_f16_resid_ln takes that plan when it is given a workspace,
 * and then leaves the workspace untouched.                                                                                    */
#define VLFM_EPI_CLUSTER_SPLIT 256
/* The cluster-split plan of an M x N x K GEMM that allows it: tile width *bn, cluster size *splits, and the bytes the busiest CTA
 * loads (*cta_bytes: K-loop operands plus the peers' partials); all zero when the shape does not take that path.          */
int vlfm_gemm_csplit_plan(int M, int N, int K, int* bn, int* splits, double* cta_bytes);

/* PIL-exact antialiased bicubic resize (uint8) + ToTensor + Normalize, emitted in the
 * im2col layout of the patch-embedding GEMM.  Replaces lavis' BlipImageEvalProcessor as
 * called at vlfm/vlm/blip2itm.py:48-49.
 * d_img [B,H,W,3] uint8; d_mid [B,H,OW,3] uint8 scratch; d_out [B*(OH/patch)*(OW/patch), ldk] fp16.
 * (h|v)bounds [2*O] = {first input index, tap count}; (h|v)kk [O*ksize] 22-bit fixed point
 * coefficients (Pillow precompute_coeffs / normalize_coeffs_8bpc). h_mean3/h_std3: HOST float[3]. */
int vlfm_preprocess_im2col(const uint8_t* d_img, uint8_t* d_mid, void* d_out, int B, int H, int W, int OH,
                           int OW, int patch, int ldk, const int32_t* d_hbounds, const int32_t* d_hkk,
                           int hksize, const int32_t* d_vbounds, const int32_t* d_vkk, int vksize,
                           const float* h_mean3, const float* h_std3, void* stream);
/* x[b,0] = cls + pos[0]; x[b,1+p] = patch[b,p] + pos[1+p]   (fp32; ViT token assembly) */
int vlfm_assemble_tokens(const float* d_patch, const float* d_cls, const float* d_pos, float* d_x, int B,
                         int T, int D, void* stream);
/* LayerNorm over the last dimension: fp32 in, fp16 (d_out16) and/or fp32 (d_out32) out. */
int vlfm_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out16, float* d_out32,
                   int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream);
/* softmax(scale * Q K^T) V per (batch, head); fp16 in/out, fp32 accumulate.
 * q rows (b*Nq + i), k/v rows (b*Nk + j), head h at column offset h*hd. Nk <= 272, hd <= 96. */
int vlfm_attention_f16(const void* d_q, const void* d_k, const void* d_v, void* d_o, int B, int heads, int Nq,
                       int Nk, int hd, int ldq, int ldk, int ldv, int ldo, float scale, void* stream);
/* ---- "x2" path: float32-grade Q-Former on the fp16 tensor path.  The reference runs the Q-Former in float32 (lavis casts
 * only the ViT to half); fp16 operands there alone move the ITC cosine by ~3e-5 (measured on the fp32 oracle), the ViT's by 1e-6.
 * An x2 operand is a pair of fp16 arrays (hi, lo) with value = hi + lo / 2048, hi = fp16(v), lo = fp16((v - hi) * 2048).
 * vlfm_gemm_f16x2: out = epilogue(A @ W^T + bias), A and W x2 operands, three wgmma per K step into two register
 *   accumulators (hi.hi | lo.hi + hi.lo).  epilogue: VLFM_EPI_BIAS_F32, VLFM_EPI_BIAS_RESID_F32, VLFM_EPI_BIAS_GELU_F16X2 (GELU, output
 *   written as x2 operands d_out / d_out_lo).
 * vlfm_gemm_f16x2_resid_ln: x += ...; LayerNorm(x) -> x2 operands (+ fp32), deterministic split-K like vlfm_gemm_f16_resid_ln.
 * vlfm_layernorm_x2 / vlfm_layernorm_reduce_x2: LayerNorm with x2 operand output.
 * vlfm_attention_f32: softmax(scale * Q K^T) V in float32 (q, k, v fp32; hd in {32, 64}; Nk <= 272), output as x2 operands.
 * vlfm_split_x2: x2 operands of an fp32 array (d_hi may be NULL when the fp16 rounding already exists). */
#define VLFM_EPI_BIAS_GELU_F16X2 6
int vlfm_gemm_f16x2(const void* d_A_hi, const void* d_A_lo, const void* d_W_hi, const void* d_W_lo, const float* d_bias, void* d_out,
                    void* d_out_lo, int M, int N, int K, int lda, int ldw, int ldo, int epilogue, void* stream);
int vlfm_gemm_f16x2_resid_ln(const void* d_A_hi, const void* d_A_lo, const void* d_W_hi, const void* d_W_lo, const float* d_bias,
                             float* d_x, int M, int N, int K, int lda, int ldw, int ldx, const float* d_gamma, const float* d_beta,
                             void* d_out_hi, void* d_out_lo, int ld16, float* d_out32, int ld32, float eps, float* d_partials,
                             size_t partial_bytes, void* stream);
int vlfm_layernorm_x2(const float* d_x, const float* d_gamma, const float* d_beta, void* d_out_hi, void* d_out_lo, float* d_out32,
                      int rows, int D, int ldx, int ldo16, int ldo32, float eps, void* stream);
int vlfm_layernorm_reduce_x2(float* d_x, const float* d_partials, int splits, long long split_stride, const float* d_gamma,
                             const float* d_beta, void* d_out_hi, void* d_out_lo, float* d_out32, int rows, int D, int ldx, int ldo16,
                             int ldo32, float eps, void* stream);
int vlfm_split_x2(const float* d_src, void* d_hi, void* d_lo, long long n, void* stream);
int vlfm_attention_f32(const float* d_q, const float* d_k, const float* d_v, void* d_o_hi, void* d_o_lo, int B, int heads, int Nq,
                       int Nk, int hd, int ldq, int ldk, int ldv, int ldo, float scale, void* stream);
/* ITC head (match_head="itc"): cos[b] = max_q <normalize(proj[b,q,:]), text>.
 * vlfm_itc_head_multi: the same against P prompts, text [P, D] (rows L2-normalised) -> out[b * ldo + p]; one launch, the
 * query norms computed once.  Column p is bitwise equal to vlfm_itc_head on text[p] (vlfm_itc_head is the P = 1 case).
 * VLFM_E_INVALID for NULL pointers, B < 1, P < 1 or ldo < P. */
int vlfm_itc_head(const float* d_proj, const float* d_text, float* d_out, int B, int Q, int D, void* stream);
int vlfm_itc_head_multi(const float* d_proj, const float* d_text, float* d_out, int B, int P, int Q, int D, int ldo, void* stream);

/* ----------------------------------------------- GroundingDINO Swin-T backbone ---- */
/* Replaces the image branch of groundingdino's predict() up to the backbone feature maps
 * (reference call site vlfm/vlm/grounding_dino.py:52-67).  GEMMs / LayerNorms reuse
 * vlfm_gemm_f16 / vlfm_layernorm.
 * vlfm_swin_patch_im2col: uint8 [B,H,W,3] -> to_tensor + ImageNet normalise (grounding_dino.py:53-54)
 *   -> fp16 [B*ceil(H/4)*ceil(W/4), 48] rows of the 4x4/4 patch-embedding GEMM.
 * vlfm_swin_window_attention: (shifted) 7x7-window attention, head_dim 32, with relative position
 *   bias [169, heads] and the SW-MSA region mask; qkv [B*H*W, 3C] fp16 -> out [B*H*W, C] fp16.
 * vlfm_swin_patch_merge: [B,H,W,C] fp32 -> [B*ceil(H/2)*ceil(W/2), 4C] fp32 (2x2 gather). */
int vlfm_swin_patch_im2col(const uint8_t* d_img, void* d_out, int B, int H, int W, const float* h_mean3,
                           const float* h_std3, void* stream);
int vlfm_swin_window_attention(const void* d_qkv, const float* d_qkv_bias, const float* d_rel_bias, void* d_out, int B,
                               int H, int W, int C, int heads, int shift, void* stream);
int vlfm_swin_patch_merge(const float* d_x, float* d_out, int B, int H, int W, int C, void* stream);

/* Confidence-cone template of ValueMap (`_get_confidence_mask` / `_get_blank_cone_mask`, value_map.py:321-355): the
 * cv2.ellipse filled sector (+-fov/2 about +row, integer degrees, OpenCV's sine table and 16.16 edge scan) times
 * remap(cos^2(remap(atan2(|dcol|,|drow|), 0, fov/2, 0, pi/2)), 0, 1, min_conf, 1).  d_out [R,R] f32, R = 2*int(max_depth*ppm)+1.
 * d_scratch needs R*R + 8*R*ceil(R/32) + 2304 bytes.  Configuration-time constant (synchronises the stream). */
int vlfm_value_cone_template(double fov, double max_depth, int ppm, double min_conf, float* d_out, void* d_scratch,
                             size_t scratch_bytes, void* stream);

/* ------------------------------------- GroundingDINO feature enhancer / decoder ---- */
/* Multi-scale deformable attention (replaces groundingdino's third-party ms_deform_attn_cuda.cu, reached from
 * vlfm/vlm/grounding_dino.py:61-67): softmax over the levels*points logits, sampling-location arithmetic
 * (MSDeformAttn.forward: loc = ref + off / (W_l, H_l) for 2-d reference points, ref_xy + off / points * ref_wh * 0.5 for
 * 4-d boxes) and the bilinear gather (zero padding, align_corners=False) in one kernel.  d_value16 [B,S,heads,32] fp16
 * (S = sum H_l*W_l, levels concatenated); d_offlog [B*Q, ld] fp32 rows holding
 * the sampling-offset projection at column 0 (heads*levels*points*2) and the attention logits at column `logit_col`
 * (heads*levels*points); d_ref [B,Q,levels,ref_dim] fp32; d_out16 [B*Q, heads*32] fp16.  head_dim 32, levels*points <= 16.
 * h_shapes_hw: HOST int32 [levels*2] = (H_l, W_l). */
int vlfm_msda_fused(const void* d_value16, const float* d_offlog, int ld, int logit_col, const float* d_ref, int ref_dim,
                    void* d_out16, int B, int S, int Q, int heads, int levels, int points, const int32_t* h_shapes_hw,
                    void* stream);
/* softmax(scale * q k^T) v per (batch, head) for head_dim 256 -- both directions of GroundingDINO's fusion-layer
 * BiMultiHeadAttention (image<-text: few keys, one chunk; text<-image: thousands of keys split into `key_chunk`-sized chunks over
 * CTAs and merged) -- or head_dim 32 (decoder self-attention over the 900 queries and text cross-attention).
 * q [B*Nq, ldq], k [B*Nk, ldk], v [B*Nk, ldv] fp16, head h at column h*head_dim; d_out16 [B*Nq, ldo] fp16.  key_chunk: multiple
 * of 16, <= 192 (head_dim 256) / <= 1024 (32).  d_part (needed when Nk > key_chunk):
 * B*heads*ceil(Nk/key_chunk)*ceilR(Nq)*(head_dim+2) floats, R = 64 / 128. */
int vlfm_biattn_f16(const void* d_q, const void* d_k, const void* d_v, void* d_out16, float* d_part, size_t part_floats, int B,
                    int heads, int head_dim, int Nq, int Nk, int ldq, int ldk, int ldv, int ldo, int key_chunk, float scale,
                    void* stream);
/* fp32 -> fp16 (round to nearest even) staging of GEMM operands. */
int vlfm_cast_f32_f16(const float* d_in, void* d_out16, long n, void* stream);
/* out_x16 = fp16(x), out_xp16 = fp16(x + pos) (query/key = hidden + position embedding); n % 4 == 0; either output may be NULL. */
int vlfm_cast_addpos_f16(const float* d_x, const float* d_pos, void* d_out_x16, void* d_out_xp16, long n, void* stream);

/* ------------------------------------------------- GroundingDINO model-level glue ---- */
/* The parts of groundingdino's `model(image, captions=[caption])` (vlfm/vlm/grounding_dino.py:61-67) that sit between the
 * backbone and the (boxes, logits) pair and outside the encoder / decoder layers (vlm/gdino_forward.py; module graph:
 * HF GroundingDinoModel.forward / GroundingDinoForObjectDetection.forward).
 * groupnorm_rows: torch.nn.GroupNorm of the neck on NHWC rows y [B,HW,C] -> d_out[b, row_off + i, :] of a [B,S,C] buffer.
 * im2col3x3s2: rows [B,h,w,C] fp32 -> fp16 [B*ho*wo, 9*C] ((ky,kx,c) order) for the fourth level's 3x3 stride-2 conv.
 * mask_rows_f16: fp32 rows -> fp16 GEMM operand with invalid rows zeroed (generate_encoder_output_proposals).
 * proposal_scores: score[b,s] = max_t <q[b,s,:], text[b,t,:]> (encoder_output_class_embed + max(-1)).
 * topk_rows: indices of the k best scores per image, descending, ties to the lower index (torch.topk; one-block bitonic sort for S <= 16384, radix select + sort of the k winners above, k <= 16384).
 * gather_rows: dst[b,i,:] = src[b, idx[b,i], :] (torch.gather).
 * box_finish: sigmoid(delta + logit(ref, eps=1e-5)).   contrastive_sigmoid: sigmoid(<hs, text>) padded with 0 to L.       */
int vlfm_groupnorm_rows(const float* d_y, int B, int HW, int C, int groups, const float* d_gamma, const float* d_beta, float eps,
                        float* d_out, int row_off, int S, void* stream);
int vlfm_im2col3x3s2(const float* d_x, void* d_col16, int B, int h, int w, int C, void* stream);
int vlfm_mask_rows_f16(const float* d_x, const uint8_t* d_valid, void* d_out16, long rows, int D, void* stream);
int vlfm_proposal_scores(const float* d_q, const float* d_text, int B, int S, int T, int D, float* d_scores, void* stream);
int vlfm_topk_rows(const float* d_scores, int B, int S, int k, long long* d_idx, void* stream);
/* decoder_query_pos: per decoder layer, reference_points_input [B,nq,L,4] = ref * (valid ratio pairs) and the sine embedding of its
 * level-0 slice (GroundingDinoDecoder.forward + get_sine_pos_embed) as the fp16 operand [B*nq, 4*P] of reference_points_head. */
int vlfm_decoder_query_pos(const float* d_ref, const float* d_valid_ratios, const float* d_dim_t, int B, int nq, int L, int P,
                           float* d_ref_in, void* d_embed16, void* stream);
int vlfm_gather_rows(const float* d_src, const long long* d_idx, int B, int S, int K, int C, float* d_dst, void* stream);
int vlfm_box_finish(const float* d_delta, const float* d_ref, float* d_out, long n, void* stream);
int vlfm_contrastive_sigmoid(const float* d_hs, const float* d_text, int B, int Q, int T, int D, int L, float* d_out, void* stream);

/* ------------------------------------------------------------- explore half ---- */
/* Replaces ObstacleMap.update_map's explore half (vlfm/mapping/obstacle_map.py:114-153) and _get_frontiers
 * (:155-169) including the two third-party frontier_exploration functions they call (spec:
 * oracle/explore_oracle.py).  One environment per call.
 * d_explored / d_nav [G,G] uint8; agent cell (col,row) = _xy_to_px(tf[:2,3]); heading_deg =
 * rad2deg(wrap(yaw + pi/2)); fov_deg = rad2deg(topdown_fov); max_line_len = max_depth*ppm;
 * area_thresh_px = area_thresh*ppm^2; nav_half = half-size of the window in which the navigable map changed.
 * d_frontiers [4096,2] float64 (x=col, y=row), d_count int32, d_status int32 (non-zero: a scratch buffer overflowed).
 * The agent may be anywhere: near the map edge the cone and the occlusion rays are clipped with cv2's own rules
 * (clipLine before every line walk, PolyEdges from clipped end points, thick segments clipped to the grid + 2 px). */
int vlfm_explore_workspace_bytes(int G, size_t* bytes);
int vlfm_explore_update(int G, uint8_t* d_explored, const uint8_t* d_nav, int agent_col, int agent_row, double heading_deg,
                        double fov_deg, double max_line_len, double area_thresh_px, int nav_half, double* d_frontiers,
                        int32_t* d_count, void* d_workspace, int32_t* d_status, void* stream);

/* The same step for a BATCH of environments in one launch sequence (every kernel runs with gridDim.y = batch).
 * frame = {col0, row0, col1, row1}: the grid rectangle ("S frame") in which the whole-grid operations of the reference
 * (explored &= navigable, component selection, frontier search) are carried out.  It must contain every cell any obstacle /
 * explore update of the episode has touched plus a margin of >= 8 cells, and each side must either be a grid edge or lie
 * >= ceil(area_thresh_px / (G - 1)) + 2 cells inside it: outside the frame explored == 0 and navigable == 1 then, which
 * makes the restriction exact (DESIGN.md section 3.2b).  {0, 0, G, G} is always valid.                                  */
typedef struct {
  int32_t slot;                 /* index of this environment's grids in d_explored / d_nav [nslots, G, G] */
  int32_t agent_col, agent_row;
  int32_t frame[4];
  int32_t pad;
  double heading_deg, fov_deg, max_line_len, area_thresh_px;
} VlfmExploreEnv;
size_t vlfm_explore_env_record_bytes(void);   /* bytes of page-locked staging per environment (h_pinned below) */
int vlfm_explore_batch_workspace_bytes(int G, int batch, size_t* bytes);
/* h_envs: host array [batch].  d_frontiers [batch,4096,2] float64, d_count / d_status [batch] int32 (call order).
 * h_pinned (optional, page-locked, >= batch * vlfm_explore_env_record_bytes()): staging for the per-environment device
 * records; it must not be reused before the copy issued by this call has executed.  Without it the records are copied
 * from pageable memory, which makes cudaMemcpyAsync wait for the stream.                                                 */
int vlfm_explore_update_batch(int G, int batch, const VlfmExploreEnv* h_envs, uint8_t* d_explored, const uint8_t* d_nav,
                              double* d_frontiers, int32_t* d_count, int32_t* d_status, void* d_workspace,
                              size_t workspace_bytes, void* h_pinned, size_t h_pinned_bytes, void* stream);
/* The two halves of vlfm_explore_update_batch: `prepare` (host only) writes the per-environment device records into h_records
 * (page-locked, >= batch * vlfm_explore_env_record_bytes()); `launch` uploads them and issues the launch sequence, whose geometry
 * depends on `batch` only -- a caller can capture `launch` once in a CUDA graph and, every step, run `prepare` + replay.        */
int vlfm_explore_prepare_batch(int G, int batch, const VlfmExploreEnv* h_envs, uint8_t* d_explored, const uint8_t* d_nav,
                               double* d_frontiers, int32_t* d_count, int32_t* d_status, void* d_workspace, size_t workspace_bytes,
                               void* h_records, size_t h_records_bytes);
int vlfm_explore_launch_batch(int G, int batch, void* d_workspace, const void* h_records, void* stream);
/* fill_small_holes for a batch of depth images [batch,H,W] -> d_filled [batch,H,W]; d_status [batch] sticky overflow flags. */
int vlfm_holes_batch_workspace_bytes(int H, int W, int batch, size_t* bytes);
int vlfm_fill_small_holes_batch(const float* d_depth, int H, int W, int batch, double area_thresh, uint8_t* d_filled,
                                void* d_workspace, size_t workspace_bytes, int32_t* d_status, void* h_pinned,
                                size_t h_pinned_bytes, void* stream);

/* -------------------------------------------------------- object point clouds ---- */
/* Replaces ObjectPointCloudMap._extract_object_cloud (vlfm/mapping/object_point_cloud_map.py:143-163) up to the random
 * subsample: cv2.erode(mask*255, None, iterations=k) (:153-154), depth 0 -> 1 -> metres in float32 (:156-158),
 * get_point_cloud (vlfm/utils/geometry_utils.py:216-236): d_points [cap,3] float64 (z, -x, -y) in np.where (row-major)
 * order, *d_count = number of mask pixels after the erosion (may exceed cap).  d_scratch >= H*W + 8*H + 512 bytes.  */
int vlfm_object_cloud_extract(const float* d_depth, const uint8_t* d_mask, int H, int W, int erosion_iterations,
                              float depth_scale, float depth_offset, double fx, double fy, double* d_points, int cap,
                              int32_t* d_count, void* d_scratch, size_t scratch_bytes, void* stream);
/* Replaces open3d_dbscan_filtering (:192-219; Open3D cluster_dbscan(eps, min_points), largest non-noise cluster, input
 * order; spec: oracle/object_map_oracle.py::dbscan_labels).  d_gather (int32[n]) or NULL: optional index list applied to
 * d_points first (the host's np.random.choice subsample, :246-266), staged in d_gathered [n,3].  n <= 65535.        */
int vlfm_dbscan_workspace_bytes(int n, size_t* bytes);
int vlfm_dbscan_largest_cluster(const double* d_points, const int32_t* d_gather, int n, double eps, int min_points,
                                double* d_gathered, double* d_out, int32_t* d_out_count, void* d_workspace,
                                size_t workspace_bytes, void* stream);

/* --------------------------------------------------------------- map frames ---- */
/* ValueMap.visualize / ObstacleMap.visualize (vlfm/mapping/value_map.py:189-219, obstacle_map.py:171-193) and the trajectory /
 * marker overlay (vlfm/mapping/traj_visualizer.py) for a batch of environments.  Frames d_out / d_frames are
 * [batch, G, G, 3] uint8 BGR, C-contiguous.  Bad arguments return VLFM_E_INVALID and launch nothing.
 *
 * vlfm_render_value: d_reduced [batch, G, G] float32 (reduced_f64 = 0) or float64 (1), call order; d_explored [nslots, G, G]
 * uint8 or NULL, row i reads slot d_slots[i] (or i when d_slots is NULL); d_lut [256, 3] uint8 (cv2 COLORMAP_INFERNO).
 * Cells with explored == 0 are zeroed, the map is flipped vertically, zero cells are white and the others take
 * lut[uint8(((v - lo) / (hi - lo)) * 255)] computed in the map's dtype with one rounding per operation (lo / hi: min / max
 * after the zero cells are set to the max; index 0 when hi == lo).  Two launches. */
int vlfm_render_workspace_bytes(int batch, size_t* bytes);
int vlfm_render_value(int G, int batch, const int32_t* d_slots, const void* d_reduced, int reduced_f64, const uint8_t* d_explored,
                      const uint8_t* d_lut, uint8_t* d_out, void* d_workspace, size_t workspace_bytes, void* stream);
/* vlfm_render_obstacle: obstacle / navigable / explored grids [nslots, G, G] uint8, frontier midpoints [nslots, max_frontiers, 2]
 * float64 (x = col, y = row) and counts [nslots] int32 as ObstacleMapBatch holds them (row i reads slot d_slots[i]).  White,
 * explored (200, 255, 200), nav == 0 the padding colour, obstacles black, frontier circles (radius 5, thickness 2,
 * (200, 0, 0)) at int() of each midpoint, then flipped vertically.  Two launches. */
int vlfm_render_obstacle(int G, int batch, const int32_t* d_slots, const uint8_t* d_obst, const uint8_t* d_nav, const uint8_t* d_explored,
                         const double* d_frontiers, const int32_t* d_count, int max_frontiers, int pad_b, int pad_g, int pad_r,
                         uint8_t* d_out, void* stream);
/* vlfm_render_draw: draws each environment's ordered list of primitives onto its frame, with the pixels of
 * cv2.line / cv2.circle (LINE_8, shift 0), clipping included.  h_lists (host, page-locked for an asynchronous upload) =
 * offsets [batch + 1] (offsets[0] = 0, non-decreasing) followed by offsets[batch] records of VLFM_DRAW_RECORD_INTS int32:
 *   {VLFM_DRAW_LINE,   x0, y0, x1, y1, 0,      thickness 1..16,         B | G << 8 | R << 16}
 *   {VLFM_DRAW_CIRCLE, cx, cy, 0,  0,  radius 0..255, thickness -1 (filled) or 1..16, colour}
 * with |coordinates| < 2^24.  list_ints = batch + 1 + 8 * offsets[batch]; the list is copied to d_lists (>= list_ints ints)
 * with one cudaMemcpyAsync on `stream`, so h_lists must not be reused before that copy has executed.  One launch. */
#define VLFM_DRAW_LINE 0
#define VLFM_DRAW_CIRCLE 1
#define VLFM_DRAW_RECORD_INTS 8
int vlfm_render_draw(int G, int batch, uint8_t* d_frames, const int32_t* h_lists, size_t list_ints, int32_t* d_lists,
                     size_t d_list_ints, void* stream);

/* ------------------------------------------------------------------ MobileSAM ---- */
/* Replaces MobileSAM.segment_bbox (vlfm/vlm/sam.py:40-57: SamPredictor.set_image + predict(box, multimask_output=False)) with the
 * TinyViT-5M encoder and the box-prompted mask decoder (engine: vlfm_b200/vlm/sam_engine.py).  GEMMs, LayerNorms and the 7-key
 * attentions run on vlfm_gemm_f16 / vlfm_gemm_f16_resid_ln / vlfm_layernorm / vlfm_attention_f16; these are the rest.
 *
 * vlfm_sam_preprocess: ResizeLongestSide(S): Pillow-exact bilinear resize [B,H,W,3] uint8 -> (OH, OW) (tables as for
 *   vlfm_preprocess_im2col, built by vlm/preprocess.py::bilinear_tables), horizontal pass first into d_mid [B,H,OW,3] uint8
 *   scratch, or with v_first = 1 (Pillow's order for frames more than 100x taller than wide that shrink vertically, see
 *   vlm/preprocess.py::pillow_vertical_first) vertical first into d_mid [B,OH,W,3]; then (x - mean) / std in fp32 (h_mean3 / h_std3: HOST float[3] on the 0..255 scale) and a zero pad to S x S -> d_out [B,S,S,3] fp16.
 * vlfm_sam_im2col3x3: fp16 NHWC [B,H,W,C] -> fp16 [B*Ho*Wo, ldk] rows of a 3x3 conv (pad 1, stride 1 or 2), column (ky*3+kx)*C + c,
 *   columns >= 9*C zero.  ldk % 8 == 0.
 * vlfm_sam_dwconv3x3: depthwise 3x3 conv (pad 1, stride 1 or 2), NHWC, weights d_w [9, C] (tap-major, BatchNorm folded) + d_b [C],
 *   then GELU when gelu != 0.  Input and output are fp32 (flag 1) or fp16 (0).
 * vlfm_sam_add_act: out = act(a + b) over n elements (b may be NULL; act = GELU when gelu != 0) -> d_out32 and / or d_out16.
 * vlfm_sam_window_attention: TinyViT window attention, head dim 32 (C = heads * 32), window ws in {7, 14}.  d_qkv [B*H*W, 3C] fp16
 *   with columns [q | k | v], head h at h*32 inside each; d_pad_qkv [3C] fp16: the q/k/v row of a padding token (the map is
 *   zero-padded to a window multiple before the attention's LayerNorm, so padded tokens are unmasked keys with this value);
 *   d_bias [heads, ws*ws] fp32 indexed by |dy|*ws + |dx|.  d_out [B*H*W, C] fp16.
 * vlfm_sam_box_tokens: decoder input tokens [M*7, D] fp32: rows 0..4 = d_fixed rows 0..4 (iou token, mask tokens), rows 5, 6 = the
 *   random-Fourier encoding of the box corners (d_boxes [M,4] float64 x1,y1,x2,y2 in frame pixels, scaled to (newh, neww) in
 *   float64, cast to float32, +0.5, / S; d_gauss [2, D/2]) plus d_fixed rows 5, 6 (corner embeddings).
 * vlfm_sam_add_pe_f16: out16 = fp16(x), outp16 = fp16(x + pe[row % pe_rows]) over [rows, D]; either output may be NULL.
 * vlfm_sam_decoder_init: d_keys [M, HW, D] = d_emb[d_frame[m]] + d_nomask (NaN rows for a frame index outside [0, F)).
 * vlfm_sam_t2i_attention: softmax(scale q k^T) v per (box, head), head dim 16, Nq <= 8 queries per box, Nk keys per box; keys are
 *   split over CTAs in 256-key chunks whose (max, sum, acc) go to d_part (M*heads*ceil(Nk/256)*Nq*18 floats) and are merged in
 *   chunk order by a second launch: bitwise reproducible, no atomics.
 * vlfm_sam_pixel_shuffle2: d_in [B*h*w, 4*C] fp32 (column (dy*2+dx)*C + c: the GEMM of a 2x2 stride-2 transposed conv)
 *   -> d_out [B, 2h, 2w, C].
 * vlfm_sam_mask_logits: d_logits [M, 2h, 2w] = sum_c d_hyper[m,c] * GELU(second transposed conv, d_up laid out as above).
 * vlfm_sam_mask_finish: low-res logits [M, L, L] -> bilinear (align_corners=False) to S x S -> crop [:newh, :neww] -> bilinear
 *   to (H, W) -> > 0 -> d_out [M, H, W] uint8. */
int vlfm_sam_preprocess(const uint8_t* d_img, uint8_t* d_mid, void* d_out, int B, int H, int W, int OH, int OW, int S,
                        const int32_t* d_hbounds, const int32_t* d_hkk, int hksize, const int32_t* d_vbounds, const int32_t* d_vkk,
                        int vksize, int v_first, const float* h_mean3, const float* h_std3, void* stream);
int vlfm_sam_im2col3x3(const void* d_x16, void* d_col16, int B, int H, int W, int C, int stride, int ldk, void* stream);
int vlfm_sam_dwconv3x3(const void* d_in, int in_f32, const float* d_w, const float* d_b, void* d_out, int out_f32, int B, int H, int W,
                       int C, int stride, int gelu, void* stream);
int vlfm_sam_add_act(const float* d_a, const float* d_b, float* d_out32, void* d_out16, long long n, int gelu, void* stream);
int vlfm_sam_window_attention(const void* d_qkv, const void* d_pad_qkv, const float* d_bias, void* d_out, int B, int H, int W, int C,
                              int heads, int ws, float scale, void* stream);
int vlfm_sam_box_tokens(const double* d_boxes, int M, int H, int W, int newh, int neww, int S, const float* d_gauss, const float* d_fixed,
                        float* d_tokens, int D, void* stream);
int vlfm_sam_add_pe_f16(const float* d_x, const float* d_pe, void* d_out16, void* d_outp16, long long rows, long long pe_rows, int D,
                        void* stream);
int vlfm_sam_decoder_init(const float* d_emb, const int32_t* d_frame, const float* d_nomask, float* d_keys, int M, int F, int HW, int D,
                          void* stream);
int vlfm_sam_t2i_attention(const void* d_q, const void* d_k, const void* d_v, void* d_o, int M, int heads, int Nq, int Nk, int ldq,
                           int ldk, int ldv, int ldo, float scale, float* d_part, size_t part_floats, void* stream);
int vlfm_sam_pixel_shuffle2(const float* d_in, float* d_out, int B, int h, int w, int C, void* stream);
int vlfm_sam_mask_logits(const float* d_up, const float* d_hyper, float* d_logits, int M, int h, int w, int C, void* stream);
int vlfm_sam_mask_finish(const float* d_low, uint8_t* d_out, int M, int L, int S, int newh, int neww, int H, int W, void* stream);

/* ------------------------------------------------------------------ PointNav ---- */
/* Replaces WrappedPointNavResNetPolicy.act (vlfm/policy/utils/pointnav_policy.py:51-128): the ResNet-18 depth encoder with
 * GroupNorm and the 2-layer LSTM of 512 (engine: vlfm_b200/policy/pointnav_engine.py).  Activations are NHWC.  Each conv is an
 * im2col pass (vlfm_pointnav_depth_in, vlfm_sam_im2col3x3, vlfm_pointnav_gather_s2) plus vlfm_gemm_f16 with VLFM_EPI_BIAS_F32;
 * these are the rest.  Every reduction has a fixed order: bitwise reproducible, and independent of the other environments.
 *
 * vlfm_pointnav_depth_in: d_depth [B,H,W] fp32 -> torch "area" resize to (IH, IW) (adaptive average pooling, fp32) -> 2x2
 *   average pool -> the rows of the 7x7 stride-2 pad-3 conv: d_col16 [B*OH*OW, ldk] fp16, column ky*7 + kx, columns >= 49 zero,
 *   OH = (IH/2 - 1)/2 + 1 (OW likewise).  d_resized [B,IH,IW] fp32 (may be NULL): the resized frame.  (H, W) == (IH, IW) is the
 *   identity resize, exact.
 * vlfm_pointnav_groupnorm: GroupNorm(G) statistics per (image, group) of d_x [B,HW,C] fp32 (biased variance, eps inside the
 *   square root), then out = act(GN_a(x) + r) -> d_out32 (may alias d_r) and / or d_out16.  rmode 0: r = 0; 1: r = d_r (fp32
 *   [B,HW,C]); 2: r = GN_b(d_y) (the downsample branch, its own statistics).  act = ReLU when relu != 0.
 * vlfm_pointnav_maxpool3s2: 3x3 stride-2 pad-1 max pool (padding is -inf) of d_x [B,H,W,C] fp32 -> d_out32 and / or d_out16.
 * vlfm_pointnav_gather_s2: the rows of a 1x1 stride-2 conv: d_out16 [B*Ho*Wo, C] = d_x16 [B, 2yo, 2xo, :] fp16, C % 8 == 0.
 * vlfm_pointnav_gemv_f32: d_y[b*ldy + n] = act(sum_k d_x[b*ldx + k] d_W[n*ldw + k] + d_bias[n]) in fp32 on CUDA cores, B <= 64;
 *   W is read once for all B.  Each (b, n) is summed in an order that depends on K only (bitwise the same for any B).
 *   K, ldx, ldw multiples of 4; d_x, d_W 16-byte aligned; d_bias may be NULL.
 * vlfm_pointnav_lstm_prep: per environment b (state slot e = d_env_ids[b]; d_state [E,4,512] = [h_l0, h_l1, c_l0, c_l1]), with
 *   the state zeroed where d_masks[b] == 0: d_xin0 [B,1088] columns 512..543 = tgt_embeding(rho, cos(-theta), sin(-theta)) of
 *   d_goal [B,2]; 544..575 = the previous-action embedding (discrete: d_w_prev [5,32] row (mask ? d_prev[e] + 1 : 0), d_prev
 *   int64 [E]; else d_w_prev [32,2] @ (mask * d_prev[e]) + d_b_prev, d_prev fp32 [E,2]); 576.. = h_l0.  d_xin1 [B,1024]
 *   columns 512.. = h_l1; d_cbuf [B,1024] = [c_l0, c_l1].  (Columns 0..511 of d_xin0 are visual_fc's output.)
 * vlfm_pointnav_lstm_cell: layer 0 from d_gates [B,2048] (i, f, g, o; both biases included): c_l0' -> d_cbuf[:, :512],
 *   h_l0' -> d_xin1[:, :512].
 * vlfm_pointnav_lstm_head: layer 1 from d_gates, then the head d_w_head [4,512] + d_b_head: d_head [B,4] (may be NULL) the four
 *   outputs (logits; or mu | log_std), d_action the action (discrete: argmax, first index on ties, int64 [B]; else tanh(mu),
 *   fp32 [B,2]), also stored to d_prev[e]; d_feat [B,512] (may be NULL) = h_l1'; d_state[e] = [h_l0', h_l1', c_l0', c_l1'].
 *   d_env_ids must not repeat. */
int vlfm_pointnav_depth_in(const float* d_depth, int B, int H, int W, int IH, int IW, void* d_col16, int ldk, float* d_resized,
                           void* stream);
int vlfm_pointnav_groupnorm(const float* d_x, const float* d_gamma_a, const float* d_beta_a, int rmode, const float* d_r,
                            const float* d_y, const float* d_gamma_b, const float* d_beta_b, float* d_out32, void* d_out16, int B, int HW,
                            int C, int G, float eps, int relu, void* stream);
int vlfm_pointnav_maxpool3s2(const float* d_x, float* d_out32, void* d_out16, int B, int H, int W, int C, void* stream);
int vlfm_pointnav_gather_s2(const void* d_x16, void* d_out16, int B, int H, int W, int C, void* stream);
int vlfm_pointnav_gemv_f32(const float* d_x, int ldx, const float* d_W, int ldw, const float* d_bias, float* d_y, int ldy, int B, int N,
                           int K, int relu, void* stream);
int vlfm_pointnav_lstm_prep(const int32_t* d_env_ids, const float* d_state, const void* d_prev, int discrete, const uint8_t* d_masks,
                            const float* d_goal, const float* d_w_goal, const float* d_b_goal, const float* d_w_prev,
                            const float* d_b_prev, float* d_xin0, float* d_xin1, float* d_cbuf, int B, void* stream);
int vlfm_pointnav_lstm_cell(const float* d_gates, float* d_cbuf, float* d_xin1, int B, void* stream);
int vlfm_pointnav_lstm_head(const float* d_gates, const float* d_cbuf, const float* d_xin1, const float* d_w_head, const float* d_b_head,
                            int discrete, const int32_t* d_env_ids, float* d_state, void* d_prev, float* d_feat, float* d_head,
                            void* d_action, int B, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VLFM_B200_H_ */

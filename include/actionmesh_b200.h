/*
 * actionmesh_b200 — C ABI of the H100-native (sm_90a) Stage-I denoising hot path of ActionMesh.
 *
 * The reference (facebookresearch/actionmesh) is pure Python on top of PyTorch library kernels; it has no FFI of its
 * own.  Each entry point below therefore cites the reference *call site* whose arithmetic it replaces (paths relative
 * to the reference checkout).  The Python host side (actionmesh_b200/*.py) binds these with ctypes and mirrors the
 * reference's operator interfaces (AttentionProcessor.__call__, ActionMeshDenoiser.forward, SchedulerFlow.denoise,
 * ImageEncoder.encode_images); see INTEGRATION.md for the reference-side binding.
 *
 * Conventions
 *  - every function returns 0 on success, a negative amb error code otherwise; amb_last_error() gives the message;
 *  - plain pointers and sizes only (no torch types); all pointers are DEVICE pointers unless stated;
 *  - the caller allocates every output; the library keeps no caller memory;
 *  - every launch is asynchronous on the given cudaStream_t (passed as void*); no hidden synchronisation;
 *  - bf16 tensors are passed as const void* / void* (uint16 storage);
 *  - "ld*" arguments are row strides in ELEMENTS.
 */
#ifndef ACTIONMESH_B200_H_
#define ACTIONMESH_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AMB_ABI_VERSION 17

typedef void* amb_stream_t; /* cudaStream_t */

/* ---- plumbing -------------------------------------------------------------------------------------------------- */
const char* amb_last_error(void);
int amb_abi_version(void);
int amb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- K9: CFG combine + Euler flow step + observed-frame mask ------------------------------------------------------
 * Replaces actionmesh/scheduler/guidance.py:95-118 (aggregate_cfg) and actionmesh/scheduler/scheduler.py:238-248
 * (flow step + masked in-place write, incl. the per-step `assert unobserved.any()` D2H sync, which is dropped).
 *   v   = p[0] + sum_i scales[i] * (p[i+1] - p[i])               (fp32 arithmetic on bf16 predictions)
 *   x_f = x_f + dt_signed * v      for every frame f with frame_update[f] != 0     (x fp32, in place)
 * pred element (branch k, frame f, e) lives at pred + k*branch_stride + f*frame_stride + frame_offset + e.
 */
int amb_cfg_euler_step(float* latents, const void* pred_bf16, int n_branches, const float* scales_host,
                       float dt_signed, const uint8_t* frame_update, int n_frames, int64_t n_per_frame,
                       int64_t branch_stride, int64_t frame_stride, int64_t frame_offset, amb_stream_t stream);

/* ---- LayerNorm (affine, fp32 statistics) ---------------------------------------------------------------------------
 * Replaces diffusers FP32LayerNorm at actionmesh/model/utils/block.py:64,83,98,107 and nn.LayerNorm at
 * actionmesh/model/temporal_denoiser.py:108,239; also DinoV2's LayerNorms (transformers modeling_dinov2).
 * x: (rows, cols) bf16 or fp32 (x_fp32), y: bf16 or fp32 (y_fp32).  cols in {256, 512, 1024, 2048, 4096}.
 */
int amb_layernorm(const void* x, int x_fp32, int64_t ldx, const float* gamma, const float* beta, void* y, int y_fp32,
                  int64_t ldy, int64_t rows, int cols, float eps, amb_stream_t stream);

/* ---- small elementwise helpers -------------------------------------------------------------------------------------
 * cast: fp32 -> bf16 (latents before proj_in, temporal_denoiser.py:205-206; context before to_k/to_v).
 * timestep embedding: diffusers Timesteps(num_channels=C, flip_sin_to_cos=False, downscale_freq_shift=0) as used at
 *   temporal_denoiser.py:57-61,209-213: t_r = t[r % n_t] * (1 - mask[r]) (mask may be NULL);
 *   out[r] = [sin(t_r*w_j) | cos(t_r*w_j)], w_j = exp(-ln(1e4) * j / (C/2)).
 * add_bias_rows: y[r, :] += bias, y bf16 or fp32 (A.5: zero-context cross-attention collapses to to_out.0.bias, block.py:146).
 */
int amb_cast_f32_bf16(const float* src, void* dst_bf16, int64_t n, amb_stream_t stream);
/* patchify: im2col for DinoV2's Conv2d(3, D, P, stride P) patch embedding (HF modeling_dinov2 Dinov2PatchEmbeddings, called
 * from actionmesh/model/image_encoder.py:53): pixels (T,3,H,W) fp32 -> bf16 rows (t,py,px) x cols (c,ky,kx), zero padded to
 * kpad (multiple of 64) columns so the projection runs on amb_gemm_bf16. */
int amb_patchify(const float* pixels, void* out_bf16, int n_images, int height, int width, int patch, int kpad,
                 amb_stream_t stream);
int amb_timestep_embedding(const float* t, int n_t, const float* mask, int rows, int channels, void* out_bf16,
                           amb_stream_t stream);
int amb_add_bias_rows(void* y, int y_fp32, int64_t ldy, const float* bias, int64_t rows, int cols, amb_stream_t stream);

/* ---- image preprocessing for the DinoV2 encoder (SURVEY 8(f) rank 3; on row a2's path) -------------------------------
 * Replaces the host BitImageProcessor call at actionmesh/model/image_encoder.py:48-51 (transformers < 5, requirements.txt:10:
 * PIL bicubic resize -> centre crop -> x 1/255 -> mean/std -> CHW).  Pillow's uint8 resize is a two-pass separable integer
 * convolution (libImaging/Resample.c): int32 coefficients with 22 fractional bits, accumulator seeded with 1 << 21,
 * (acc >> 22) clamped to [0, 255], uint8 between the passes; both passes are reproduced bit-exactly.
 *  resize_h_u8: src (n, in_h, in_w, channels_in in {3,4}) u8 -> dst (n, n_rows, out_w, 3) u8 for source rows [y0, y0+n_rows);
 *    bounds (out_w, 2) = (first source column, tap count), coeffs (out_w, ksize) — host-built, already restricted to the
 *    cropped output window.  All table entries must address columns inside [0, in_w).
 *  resize_v_normalize: src as written by resize_h_u8 -> dst (n, 3, out_h, out_w) fp32 = (lut256[u8] - mean[c]) / std[c];
 *    bounds (out_h, 2) in SOURCE row numbers, every tap inside [y0, y0+n_rows); mean/std are HOST pointers to 3 floats;
 *    dst_u8 (optional, may be NULL) receives the resized+cropped uint8 image (n, out_h, out_w, 3). */
int amb_resize_h_u8(const uint8_t* src, int n_images, int in_h, int in_w, int channels_in, int y0, int n_rows,
                    const int32_t* bounds, const int32_t* coeffs, int ksize, int out_w, uint8_t* dst, amb_stream_t stream);
int amb_resize_v_normalize(const uint8_t* src, int n_images, int n_rows, int y0, int out_w, const int32_t* bounds,
                           const int32_t* coeffs, int ksize, int out_h, const float* lut256, const float* mean3_host,
                           const float* std3_host, float* dst, uint8_t* dst_u8, amb_stream_t stream);

/* ---- frame preprocessing before the encoders (SURVEY 8(f) rank 3, second half) -------------------------------------------
 * Replaces the host numpy/PIL arithmetic of ImagePreprocessor.process_images (actionmesh/preprocessing/image_processor.py:
 * 26-146): RGBA frames are composited on a white background, cropped to the (shared or per-frame) foreground bounding box
 * and padded to a square with a margin.
 *  alpha_stats: rgba (n, h, w, 4) u8 -> stats (n, 5) int32 = xmin, ymin, xmax, ymax of alpha > 0 (:57-64; xmax = -1 when the
 *    frame is fully transparent) and the number of pixels with alpha > 127 (is_valid_alpha, :15-23).
 *  composite_crop_pad: -> out (n, box_h + 2 pad_y, box_w + 2 pad_x, 3) u8.  Inside the box: the float32 composite of :44-52 in
 *    the reference's operation order, times 255, truncated like `(img * 255).astype(uint8)` (:143-145); outside: 255.
 *    The uint8 result is bit-identical to the reference's PIL output. */
int amb_alpha_stats(const uint8_t* rgba, int n_images, int height, int width, int32_t* stats, amb_stream_t stream);
int amb_composite_crop_pad(const uint8_t* rgba, int n_images, int height, int width, int box_x, int box_y, int box_w, int box_h,
                           int pad_x, int pad_y, uint8_t* out, amb_stream_t stream);

/* ---- ActionBench evaluation (SURVEY 8(f) rank 4) ----------------------------------------------------------------------
 * Replaces scipy's KDTree.query at actionbench/chamfer.py:44-50,78-82: for each of n_query points (xyz fp32, row-major) the
 * Euclidean distance to and the index of its nearest point among n_reference points.  scratch_u64: n_query * 8 bytes of
 * device memory; out_dist / out_index: either may be NULL.  Ties resolve to the lowest index. */
int amb_nearest_neighbors(const float* query, int n_query, const float* reference, int n_reference, void* scratch_u64,
                          float* out_dist, int32_t* out_index, amb_stream_t stream);

/* ---- ActionBench gradient ICP (csrc/icp.cu; SURVEY 8(f) rank 4) --------------------------------------------------------
 * Replaces the optimisation loop of gradient_icp (actionbench/icp.py:53-112) for F frames x C candidates at once (the
 * reference: one frame, C = 24).  pred: (F, P, 3) fp32, gt: (F, Q, 3) fp32.  Per (frame f, candidate n): rot (F, C, 9) = R
 * row-major; params (F, C, 12) fp32 = T (3), the 6D rotation d6 (6), s (3), in torch.optim.Adam's parameter order; the
 * prediction is y_i = (s * x_i) @ R + T (row vectors).  1 <= C <= 1024; F, P, Q >= 1.
 *  icp_scratch_doubles: the fp64 scratch icp_chamfer_grad needs for these sizes.
 *  icp_chamfer_grad: sums (F, C, 13) fp64 = the loss L = (1/P) sum_i min_j |y_i - g_j|^2 + (1/Q) sum_j min_i |y_i - g_j|^2
 *    (pytorch3d chamfer_distance, batch_reduction=None), then t = sum G (3) and A = sum x ⊗ G (3x3 row-major, over the
 *    untransformed x), where G = (2/P)(y_i - g_a(i)) for every pred point (a(i): nearest gt point) and (2/Q)(y_b(j) - g_j),
 *    paired with x_b(j), for every gt point (b(j): nearest prediction).  Ties go to the lowest index.  The result does not
 *    depend on scheduling (no float atomics).
 *  icp_adam_step: with those sums, dL/dT = t, dL/dR[k,l] = s_k A[k,l], dL/ds_k = sum_l R[k,l] A[k,l], all scaled by 1/C
 *    (the reference back-propagates the mean over candidates), back-propagated through R = rot_init (C, 9) @
 *    rotation_6d_to_matrix(d6); one torch.optim.Adam step (defaults) on params with moments adam_m, adam_v (F, C, 12) fp32,
 *    where step_size = -lr / (1 - 0.9^t) and bias2_sqrt = sqrt(1 - 0.999^t) for step t >= 1; best (F, 16) fp32 = loss, R (9),
 *    T (3), s (3) of the best candidate so far, updated as icp.py:99-106 does (init loss = +inf); rot is overwritten with R of
 *    the updated params.
 *  icp_transform_points: points (F, n_points, 3) fp32 -> out = p @ M + T with M[k,l] = s_k R[k,l] (fp32, the matrix product
 *    pytorch3d's Scale(s).compose(Rotate(R), Translate(T)).transform_points applies); transform holds R (9), T (3), s (3) of
 *    frame f at transform + f * transform_stride (stride 0: one transform for every frame).  frames <= 65535. */
int amb_icp_scratch_doubles(int frames, int candidates, int n_pred, int n_gt, int64_t* out_doubles);
int amb_icp_chamfer_grad(const float* pred, const float* gt, int frames, int candidates, int n_pred, int n_gt,
                         const float* rot, const float* params, double* scratch, double* sums, amb_stream_t stream);
int amb_icp_adam_step(const double* sums, const float* rot_init, int frames, int candidates, float step_size,
                      float bias2_sqrt, float* params, float* adam_m, float* adam_v, float* rot, float* best,
                      amb_stream_t stream);
int amb_icp_transform_points(const float* points, int frames, int64_t n_points, const float* transform,
                             int64_t transform_stride, float* out, amb_stream_t stream);

/* ---- Stage II (temporal autoencoder) helpers — first "next" row of SURVEY 8(f) -----------------------------------------
 * alpha_rows: the (source_alpha, target_alpha) token of actionmesh/model/temporal_autoencoder.py:233-237 (TimestepEmbedder,
 *   model/utils/embeddings.py:56-132), fp32, written to n_rows rows `row_stride` elements apart.
 * point_embedding: FrequencyPositionalEmbedding of the query vertices (+ normals), temporal_autoencoder.py:240-243,
 *   embeddings.py:15-53, as fp32 rows zero-padded to kpad columns for the proj_query GEMM.
 * displacement_out: 2*sigmoid(-logits) - 1 on the first out_dim columns (temporal_autoencoder.py:160,269).
 * split3_bf16 / softmax_split3: the reference runs the vertex-query cross-attention block with autocast DISABLED (fp32,
 *   temporal_autoencoder.py:264-266).  Here that block runs on the bf16 tensor cores at fp32-grade accuracy by splitting
 *   every operand x = hi + lo (two bf16) and concatenating along K: activations as [hi | lo | hi] (w_pattern = 0),
 *   weights as [hi | hi | lo] (w_pattern = 1), so one amb_gemm_bf16 call evaluates a_hi w_hi + a_lo w_hi + a_hi w_lo
 *   with fp32 accumulation.  split3_bf16 cuts `cols` in segments of `seg` columns (each becomes 3*seg output columns);
 *   softmax_split3 does the row softmax of fp32 scores (n valid columns, scaled by `scale`) and writes the probabilities
 *   as the activation split with each part n_pad wide (zeros in the padding). */
int amb_alpha_rows(float source_alpha, float target_alpha, int size, float* out, int64_t row_stride, int n_rows,
                   amb_stream_t stream);
int amb_point_embedding(const float* points, int n_points, int in_dim, int extra, int num_freqs, int include_pi,
                        float* out, int kpad, amb_stream_t stream);
int amb_displacement_out(const float* logits, int64_t ld, int n_points, int out_dim, float* out, amb_stream_t stream);
int amb_split3_bf16(const float* src, int64_t ld_src, int64_t rows, int cols, int seg, int w_pattern, void* dst_bf16,
                    int64_t ld_dst, amb_stream_t stream);
int amb_softmax_split3(const float* scores, int64_t ld_s, int rows, int n, int n_pad, float scale, void* dst_bf16,
                       int64_t ld_dst, amb_stream_t stream);

/* ---- wgmma GEMM with fused epilogues: C = epi(A · Wᵀ) ----------------------------------------------------------------
 * Replaces every nn.Linear on the path (cuBLAS in the reference): proj_in/proj_out/time_proj
 * (temporal_denoiser.py:206,213-214,242), linear_skip on cat[skip,h] without materialising the concat (block.py:131-133,
 * a2/k_split), to_q/to_k/to_v with the head split, RMS qk-norm and RoPE of attention_processor.py:92-130 fused in the
 * epilogue, to_out + residual (attention_processor.py:147, block.py:137,146), FeedForward GELU(erf) MLP (block.py:152).
 * A:(m,k) bf16 row-major, W:(n,k) bf16 row-major (nn.Linear layout), fp32 accumulation in registers.
 * k % 64 == 0, n % 64 == 0.
 */
typedef struct amb_gemm_args {
  const void* a;        /* bf16 (m, k) */
  int64_t lda;
  const void* a2;       /* optional second A source supplying columns k >= k_split (NULL = unused) */
  int64_t lda2;
  int32_t k_split;      /* multiple of 64 */
  const void* w;        /* bf16 (n, k) */
  int64_t ldw;
  void* c;              /* bf16 or fp32 (m', n) */
  int64_t ldc;
  int32_t c_fp32;
  int32_t m, n, k;
  const float* bias;    /* (n) or NULL */
  const void* residual; /* (m', n) bf16/fp32 or NULL; added after the activation; may alias c */
  int64_t ldr;
  int32_t res_fp32;
  int32_t act;          /* 0 none, 1 GELU(erf), 2 ReLU (RMBG's REBNCONV, briarmbg.py:24) */
  const float* col_scale; /* (n) or NULL: per-column scale applied after bias/act, before residual (DinoV2 LayerScale) */
  /* output row remap: dst_row = (row / grp_rows) * grp_stride + row % grp_rows + row_off  (grp_rows == 0: identity) */
  int32_t grp_rows, grp_stride, row_off;
  /* per-head (128 columns) RMSNorm for columns [0, norm_cols): weight norm_w0 for col < norm_seg, norm_w1 otherwise
   * (norm_cols may be 0 with rope_cols > 0: RoPE without q/k norm, as in the Stage-II blocks) */
  int32_t norm_cols, norm_seg;
  const float* norm_w0;
  const float* norm_w1;
  float norm_eps;
  /* interleaved-pair RoPE for columns [0, rope_cols): cos/sin tables (n_pos, 64) fp32, pos = row / rope_rows_per_pos */
  int32_t rope_cols;
  const float* rope_cos;
  const float* rope_sin;
  int32_t rope_rows_per_pos;
  /* optional second output: the same final values rounded to bf16, (m', n) row-major with row stride ldc2 (plain epilogue only).
   * Used with the fp32 residual stream: the fp32 result continues the stream, the bf16 copy is the GEMM operand of the
   * long-skip linear (block.py:131-133), so no separate cast pass is needed. */
  void* c2;
  int64_t ldc2;
} amb_gemm_args;

int amb_gemm_bf16(const amb_gemm_args* args, amb_stream_t stream);

/* ---- wgmma flash attention forward -------------------------------------------------------------------------------
 * Replaces F.scaled_dot_product_attention at actionmesh/model/utils/attention_processor.py:133-139 (non-causal, no
 * mask, dropout 0) for the inflated self-attention (S = T*(N+1)) and the per-frame cross-attention (S_k = 257), and
 * DinoV2's attention (head_dim 64).  Strided 4-D views so q/k/v are read straight out of the fused QKV GEMM output and
 * o is written in (b, s, h*d) order for to_out.  Strides in elements; the innermost (d) stride is 1.
 * kv may be split in `kv_chunks` equal chunks of `sk_chunk` keys whose base pointers are k + c*k_chunk_stride (used by
 * the frame-sharded window: chunk c is rank c's all-gathered K/V).  kv_chunks == 1 for the plain case.
 */
typedef struct amb_attn_args {
  const void* q;
  const void* k;
  const void* v;
  void* o;
  int64_t q_stride_b, q_stride_h, q_stride_s;
  int64_t k_stride_b, k_stride_h, k_stride_s;
  int64_t v_stride_b, v_stride_h, v_stride_s;
  int64_t o_stride_b, o_stride_h, o_stride_s;
  int32_t batch, heads, sq, sk, head_dim;
  float scale; /* softmax scale, 1/sqrt(head_dim) in the reference */
  int32_t kv_chunks;
  int32_t sk_chunk;
  int64_t k_chunk_stride, v_chunk_stride;
} amb_attn_args;

int amb_flash_attn_fwd(const amb_attn_args* args, amb_stream_t stream);

/* fp32 attention for short sequences, head_dim 64 (the DinoV2 encoder, which the reference runs in fp32 outside autocast:
 * actionmesh/pipeline.py:664-667, model/image_encoder.py:38-55 -> HF Dinov2SelfAttention's scaled_dot_product_attention).
 * q, k, v: fp32, element (frame f, token s, head h, d) at ptr[(f * seq + s) * ld + h * 64 + d]; out likewise with ldo.
 * seq <= 320.  No mask, non-causal; softmax(scale * q k^T) v with fp32 arithmetic throughout (CUDA cores). */
int amb_attn_small_f32(const float* q, const float* k, const float* v, int64_t ld, int frames, int seq, int heads, float scale,
                       float* out, int64_t ldo, amb_stream_t stream);

/* ---- Stage 0's anchor mesh: octree refinement + dual marching cubes (SURVEY 8(f) row f2) ------------------------------
 * Replaces flash_extract_geometry (third_party/TripoSG/triposg/inference_utils.py:318-479) after the decoder calls, and the
 * DiffDMC iso-surface extraction it hands the final grid to.  Grids are cubic with n points per side, x slowest:
 * element (x, y, z) at (x * n + y) * n + z.  Masks are uint8 0/1.
 *  octree_near_surface: mask = (a face neighbour has another sign, with replicate padding and invalid (<= -9000) neighbours
 *    replaced by the cell itself, on a valid cell) or |logit| < 0.95 (inference_utils.py:203-297,402-403).
 *  octree_dilate: out = any of the 3x3x3 zero-padded neighbourhood set (the ones-Conv3d "> 0" of :361-362,410-416).
 *  octree_mark_upsampled: fine ((2n-1)^3) = 0 except fine[2x, 2y, 2z] = coarse[x, y, z] (:414).
 *  octree_count_points / octree_emit_points: the set cells of a mask as a point list in grid order, xyz fp32 (P, 3) =
 *    fp32(idx) * resolution + bbox_min with both ops rounded separately (:417-421; resolution and bbox_min are HOST
 *    pointers to 3 floats) and the linear grid index (P).  `scratch` holds amb_scan_scratch_ints(n^3) ints; after the
 *    count, its last entry (device memory) is P.
 *  grid_fill / grid_replace / grid_scatter: g[:] = value; g[g == from] = to; g[index[i]] = values[i * ld].
 *  dmc_count / dmc_emit: dual marching cubes of the zero level set, inside = logit > 0.  cases: (n-1)^3 bytes;
 *    vertex_scratch: amb_scan_scratch_ints((n-1)^3) ints, face_scratch: amb_scan_scratch_ints(n^3) ints; after the count
 *    their last entries are V and F.  dmc_emit writes vertex_offsets ((n-1)^3 int32), vertices (V, 3) fp32 in grid-index
 *    units, faces (F, 3) int32 wound outward from the inside.  The patch table and the face rules are in csrc/geometry.cu
 *    and DESIGN.md. */
int amb_scan_scratch_ints(int64_t n_items, int64_t* out_ints);
int amb_octree_near_surface(const float* grid, int n, uint8_t* mask, amb_stream_t stream);
int amb_octree_dilate(const uint8_t* in, int n, uint8_t* out, amb_stream_t stream);
int amb_octree_mark_upsampled(const uint8_t* coarse, int n, uint8_t* fine, amb_stream_t stream);
int amb_octree_count_points(const uint8_t* mask, int n, int32_t* scratch, amb_stream_t stream);
int amb_octree_emit_points(const uint8_t* mask, int n, const int32_t* scratch, const float* resolution3_host,
                           const float* bbox_min3_host, float* xyz, int32_t* index, amb_stream_t stream);
int amb_grid_fill(float* grid, int64_t count, float value, amb_stream_t stream);
int amb_grid_replace(float* grid, int64_t count, float from, float to, amb_stream_t stream);
int amb_grid_scatter(const float* values, int64_t ld, const int32_t* index, int count, float* grid, amb_stream_t stream);
int amb_dmc_count(const float* grid, int n, uint8_t* cases, int32_t* vertex_scratch, int32_t* face_scratch,
                  amb_stream_t stream);
int amb_dmc_emit(const float* grid, int n, const uint8_t* cases, const int32_t* vertex_scratch, const int32_t* face_scratch,
                 int32_t* vertex_offsets, float* vertices, int32_t* faces, amb_stream_t stream);

/* ---- mesh input: the TripoSG VAE encoder's point sampling and posterior (csrc/point_sampling.cu) -------------------------
 *  farthest_point_sample: replaces pytorch3d's sample_farthest_points(points[..., :3], K, random_start_point=True) called by
 *    TripoSGVAE._sample_features (actionmesh/external/triposg.py:113-151, model/utils/pointcloud_sampling.py:54-62).
 *    points: fp32, point i of batch element b has its x, y, z at points + b * batch_stride + i * ld (+0, +1, +2), so the xyz
 *    of wider rows (xyz + normal) is read in place.  start: (batch) int64 DEVICE array in [0, n).  out: (batch, k) int64.
 *    out[b, 0] = start[b]; every point keeps d = min over the selected points of ((dx*dx) + (dy*dy)) + (dz*dz), fp32 with each
 *    operation rounded on its own, initialised to +inf; out[b, r] = argmax d with ties to the lowest index (once every d is
 *    0 that is index 0 again, as a plain argmax).  Deterministic.  1 <= n <= 16384.
 *  gaussian_sample: DiagonalGaussianDistribution (third_party/TripoSG/triposg/models/autoencoders/vae.py:8-36) on the fp32
 *    `quant` output (rows, >= 2C) with row stride ld: logvar = clamp(params[:, C:2C], -30, 20), std = exp(0.5 logvar),
 *    z = params[:, :C] + std * eps.  eps, z, logvar, std_out: contiguous (rows, C) fp32; any of z, logvar, std_out may be
 *    NULL (eps only needed with z). */
int amb_farthest_point_sample(const float* points, int batch, int n, int64_t ld, int64_t batch_stride, const int64_t* start,
                              int k, int64_t* out, amb_stream_t stream);
int amb_gaussian_sample(const float* params, int64_t ld, int64_t rows, int channels, const float* eps, float* z,
                        float* logvar, float* std_out, amb_stream_t stream);

/* ---- anchor-mesh post-processing: quadric edge-collapse decimation and floater removal (csrc/mesh_process.cu) -------------
 * Replaces MeshPostprocessor.process_mesh's decimation and floater removal (actionmesh/preprocessing/mesh_processor.py:
 * 104-161,288-325,374-425: trimesh simplify_quadric_decimation and split(only_watertight=False)).  The rules are in
 * csrc/mesh_process.cu and DESIGN.md §15; actionmesh_b200/mesh_process.py drives the rounds.
 * positions: (V, 3) fp64; faces: (F, 3) int32, three distinct indices in [0, V) (not checked on the device).  `scan` holds
 * amb_scan_scratch_ints(max(V, F)) ints; `work` holds V ints.  Zero vertices or faces launch nothing (collapse_select still
 * zeroes its counters).
 *  mesh_adjacency: vf_offsets (V + 1) and vf_faces (3F): each vertex's faces in ascending order; neighbours (6F): per vertex
 *    (from 2 * vf_offsets[v]) the other two corners of each of its faces, sorted.  Then counts the edges: afterwards
 *    scan[amb_scan_scratch_ints(V) - 1] (device) is E.
 *  mesh_edges (after mesh_adjacency, same scan; work receives each vertex's first edge): edges (E, 5) int32 = a < b, face count, and the (up to 2) faces holding the
 *    edge in ascending order (-1 when absent or when more than 2 faces hold it), ordered by (a, b); flags (V) = bit 0 boundary
 *    vertex, bit 1 vertex on a non-manifold edge.
 *  mesh_quadrics: quadrics (V, 10) fp64, the upper triangle of each vertex's 4x4 error quadric row by row.
 *  mesh_collapse_select: per edge its key (uint64; all ones when the collapse is invalid) and target (E, 3) fp64;
 *    vertex_min (2V) uint64 = the minimum key at each vertex, then over its 1-ring; remap (V) = identity; counters (2) =
 *    number of winning edges and the faces they would remove; winners (2E) = (key, face count) of each winner, unordered.
 *  mesh_collapse_apply: every winner with key <= key_limit collapses b into a: remap[b] = a, a moves to its target,
 *    Q_a += Q_b.
 *  mesh_compact_faces: out_faces = the faces, in order, whose corners (through remap when given) are distinct and, when
 *    labels is given, whose component has >= min_size faces (sizes[labels[f]]).  scan[last] (device) is their count.
 *  mesh_compact_vertices: the referenced vertices in index order -> out_positions, and out_faces = faces renumbered;
 *    scan[amb_scan_scratch_ints(V) - 1] (device) is their count.
 *  mesh_components: one union pass over the edges with exactly 2 faces (first != 0 initialises labels (F) to 0..F-1); *changed
 *    (device) is 0 once labels are final, each then the smallest face index of its edge-connected component.
 *  mesh_component_sizes: sizes (F) = number of faces carrying each label. */
int amb_mesh_adjacency(const int32_t* faces, int64_t n_faces, int64_t n_vertices, int32_t* work, int32_t* scan,
                       int32_t* vf_offsets, int32_t* vf_faces, int32_t* neighbours, amb_stream_t stream);
int amb_mesh_edges(const int32_t* faces, int64_t n_faces, int64_t n_vertices, const int32_t* vf_offsets,
                   const int32_t* vf_faces, const int32_t* neighbours, int32_t* work, const int32_t* scan, int32_t* edges,
                   uint8_t* flags, amb_stream_t stream);
int amb_mesh_quadrics(const double* positions, const int32_t* faces, int64_t n_vertices, const int32_t* vf_offsets,
                      const int32_t* vf_faces, const int32_t* neighbours, double* quadrics, amb_stream_t stream);
int amb_mesh_collapse_select(const double* positions, const double* quadrics, const int32_t* faces, int64_t n_vertices,
                             const int32_t* vf_offsets, const int32_t* vf_faces, const int32_t* neighbours,
                             const int32_t* edges, int64_t n_edges, const uint8_t* flags, uint64_t* keys, double* targets,
                             uint64_t* vertex_min, int32_t* remap, uint64_t* counters, uint64_t* winners,
                             amb_stream_t stream);
int amb_mesh_collapse_apply(const int32_t* edges, int64_t n_edges, int64_t n_vertices, const uint64_t* keys,
                            const double* targets, const uint64_t* vertex_min, uint64_t key_limit, int32_t* remap,
                            double* positions, double* quadrics, amb_stream_t stream);
int amb_mesh_compact_faces(const int32_t* faces, int64_t n_faces, const int32_t* remap, const int32_t* labels,
                           const int32_t* sizes, int min_size, int32_t* scan, int32_t* out_faces, amb_stream_t stream);
int amb_mesh_compact_vertices(const double* positions, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                              int32_t* work, int32_t* scan, double* out_positions, int32_t* out_faces, amb_stream_t stream);
int amb_mesh_components(const int32_t* edges, int64_t n_edges, int64_t n_faces, int first, int32_t* labels, int32_t* changed,
                        amb_stream_t stream);
int amb_mesh_component_sizes(const int32_t* labels, int64_t n_faces, int32_t* sizes, amb_stream_t stream);

/* ---- multi-view normal rendering: vertex normals, rasterization, normal-image compositing (csrc/render.cu) ------------------
 * Replaces ActionMeshVisualizer.render's per-view PyTorch3D calls (actionmesh/render/visualizer.py:109-141, renderer.py:87-185):
 * Meshes.verts_normals_packed, MeshRasterizer (naive, bin_size=0, one face per pixel, blur 0, perspective-correct, clipped
 * barycentrics, no culling, no z clip) at 2S x 2S samples, soft_normal_shading, the 2x2 average-pooled mask and
 * make_normal_image's nearest reduction and white composite.  DESIGN.md §16 gives every formula; actionmesh_b200/render.py
 * drives the calls.  All arithmetic is fp32 with each operation rounded on its own, in the order DESIGN.md states.
 * vertices: (V, 3) fp32; faces: (F, 3) int32 in [0, V) (not checked on the device).  cameras: (C, 12) fp32 DEVICE array, R
 * row-major then T, with X_view = X R + T (row vectors); focal is the focal length f, principal point 0.  V < 2^31 - 1 and
 * 6F < 2^31.
 *  render_vertex_normals: normals (V, 3) = each vertex's sum of cross(v1 - v0, v2 - v0) over its faces in ascending face order,
 *    divided by max(|n|, 1e-6).  vf_offsets / vf_faces come from amb_mesh_adjacency on the same faces (which needs three
 *    distinct corners per face).  Zero vertices launch nothing.
 *  render_rasterize: pix_to_face (C, 2S, 2S) int32 = for each sample the face with the smallest non-negative depth, ties to the
 *    lower index, -1 where none covers it.  depth_keys: C * 4 S^2 uint64 of scratch; queue: C * F + 1 int32 of scratch.
 *    C * 4 S^2 and C * F must fit int32.  Zero faces give an all -1 pix_to_face (vertices and faces may then be NULL).  The
 *    result does not depend on scheduling.
 *  render_shade_normals: for each view c and output pixel (i, j) of S x S, the uint8 RGB of the composited normal image,
 *    written at out + i * row_stride + c * view_stride + 3 j (+0, +1, +2) so the views land side by side in a grid row
 *    (strides in bytes; view_stride >= 3 S when C > 1).  pix_to_face as written by render_rasterize with the same vertices,
 *    faces, cameras, focal and S; normals as written by render_vertex_normals.  With zero faces every cell is white and
 *    vertices, faces and normals may be NULL. */
int amb_render_vertex_normals(const float* vertices, int64_t n_vertices, const int32_t* faces, const int32_t* vf_offsets,
                              const int32_t* vf_faces, float* normals, amb_stream_t stream);
int amb_render_rasterize(const float* vertices, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                         const float* cameras, int n_cameras, float focal, int image_size, uint64_t* depth_keys,
                         int32_t* queue, int32_t* pix_to_face, amb_stream_t stream);
int amb_render_shade_normals(const float* vertices, int64_t n_vertices, const int32_t* faces, int64_t n_faces,
                             const float* normals, const float* cameras, int n_cameras, float focal, int image_size,
                             const int32_t* pix_to_face, uint8_t* out, int64_t row_stride, int64_t view_stride,
                             amb_stream_t stream);

/* ---- background removal: RMBG-1.4 around split-bf16 GEMM convolutions, mask head and refinement (csrc/rmbg.cu) -------------
 * Replaces BackgroundRemover.forward (actionmesh/preprocessing/background_removal.py:84-112) with BriaRMBG
 * (third_party/TripoSG/scripts/briarmbg.py:355-463).  Every 3x3 convolution is rmbg_im2col_split followed by amb_gemm_bf16 on
 * the split operand (BN folded into the weights, act 2, the RSU residual as the GEMM residual); DESIGN.md §17 and
 * actionmesh_b200/background_removal.py drive the calls.  Activations are fp32 NHWC: pixel p, channel c at p * ps + c, with a
 * pixel stride ps >= the channel count.  Bilinear resampling is align_corners=False with scale = in / out in fp32, src =
 * max(scale (dst + 0.5) - 0.5, 0) and h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11), every operation rounded on its own.
 * Images are at most 2^30 pixels.
 *  rmbg_resize_input: uint8 RGB (height, width, 3) -> fp32 (out_height, out_width, 3) = bilinear / 255 - 0.5 (_preprocess_image,
 *    background_removal.py:57-69).
 *  rmbg_im2col_split: the 3x3 patches (stride 1 or 2, dilation d, padding <= d) of the channel concatenation [src0 | src1]
 *    (src1 NULL when c1 = 0; replaces the RSU decoders' torch.cat, briarmbg.py:99-114) -> bf16 rows (out_h * out_w, ld_dst)
 *    with columns (ky, kx, c) zero-padded to k_pad (a multiple of 64), written as amb_split3_bf16's activation layout
 *    [hi | lo | hi] with seg = k_pad.  out_h = (height + 2 pad - 2 d - 1) / stride + 1.
 *  rmbg_maxpool2: MaxPool2d(2, stride=2, ceil_mode=True) (briarmbg.py:49) -> (ceil(h / 2), ceil(w / 2), channels).
 *  rmbg_upsample: _upsample_like (briarmbg.py:29-33) to (out_height, out_width).
 *  rmbg_mask_head: side1 (3x3, 64 -> 1, bias; weight = 576 fp32 in (ky, kx, c) order, then the bias) on the stage1d features
 *    -> logits (height, width); soft = sigmoid(upsample(logits)) at the model size (result[0][0], briarmbg.py:445-446,463);
 *    resized = upsample(soft) at the frame size, and mask = uint8((resized - min) / (max - min) * 255), truncated
 *    (_postprocess_mask, background_removal.py:71-82).  When max == min the reference divides by zero; mask is then all 0.
 *    minmax: 2 int32 of scratch.  feat 16-byte aligned with ps >= 64, a multiple of 4.
 *  rmbg_refine_rgba: rgba (height, width, 4) = the RGB frame with alpha = mask (refine 0) or refine_mask(mask, min_size)
 *    (refine 1, background_removal.py:20-38): cv2's Otsu threshold t (in double, as OpenCV computes it), foreground mask > t,
 *    8-connected components, components of fewer than min_size pixels dropped, 0 / 255.  hist: 257 int32 (the histogram, then
 *    t); labels, sizes: height * width int32 (each foreground pixel's component root = its smallest pixel index, and each
 *    root's pixel count).  The result does not depend on scheduling.
 */
int amb_rmbg_resize_input(const uint8_t* rgb, int height, int width, float* out, int out_height, int out_width,
                          amb_stream_t stream);
int amb_rmbg_im2col_split(const float* src0, int c0, int64_t ps0, const float* src1, int c1, int64_t ps1, int height, int width,
                          int stride, int pad, int dilation, int k_pad, void* dst_bf16, int64_t ld_dst, amb_stream_t stream);
int amb_rmbg_maxpool2(const float* src, int64_t ps_src, int height, int width, int channels, float* dst, int64_t ps_dst,
                      amb_stream_t stream);
int amb_rmbg_upsample(const float* src, int64_t ps_src, int height, int width, int channels, float* dst, int64_t ps_dst,
                      int out_height, int out_width, amb_stream_t stream);
int amb_rmbg_mask_head(const float* feat, int64_t ps, int height, int width, const float* weight, float* logits, int model_height,
                       int model_width, float* soft, int out_height, int out_width, float* resized, int32_t* minmax,
                       uint8_t* mask, amb_stream_t stream);
int amb_rmbg_refine_rgba(const uint8_t* rgb, const uint8_t* mask, int height, int width, int refine, int min_size,
                         int32_t* hist, int32_t* labels, int32_t* sizes, uint8_t* rgba, amb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ACTIONMESH_B200_H_ */

/* painter_b200 — C ABI of the H100-native Painter/SegGPT hot path.
 *
 * The reference (baaivision/Painter) has no FFI layer: its hot path is the Python module
 * Painter/models_painter.py (+ SegGPT/SegGPT_inference/models_seggpt.py, util/vitdet_utils.py), every
 * arithmetic step being a torch op.  Each entry point below replaces one group of those torch call
 * sites (cited per function) with a hand-written sm_90a kernel.  The host-side mirror of the
 * reference nn.Module API (painter_b200/models_painter.py, models_seggpt.py) calls these through
 * ctypes; see INTEGRATION.md for the binding.
 *
 * Conventions
 *  - all pointers are DEVICE pointers owned by the caller (PyTorch's caching allocator); the library
 *    never allocates device memory and keeps no pointer past return;
 *  - `stream` is a cudaStream_t passed as void*; kernels are enqueued asynchronously on it;
 *  - return value 0 = ok; otherwise pk_last_error() describes the failure (thread-local);
 *  - bf16 = raw 16-bit bfloat16, f32 = IEEE float. "tokens" are rows of [B*h*w, C] matrices.
 */
#ifndef PAINTER_B200_H
#define PAINTER_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int pk_version(void);
const char* pk_last_error(void);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches claim) */
long long pk_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Dense contraction on the tensor cores (wgmma):  C[M,N] = A[M,K] . B[N,K]^T   (bf16 x bf16 -> fp32)
 * Replaces every nn.Linear / F.linear on the path (models_painter.py:60-61,76,87 qkv/proj; timm Mlp
 * fc1/fc2 used at :201; decoder_embed :327,423) and their autograd backward (dgrad / wgrad GEMMs).
 *   transA = 0: A stored [M,K] row-major (lda = row stride, elements)   transA = 1: stored [K,M]
 *   transB = 0: B stored [N,K] row-major (ldb)                          transB = 1: stored [K,N]
 * Epilogues (PkEpilogue.kind):
 */
enum {
  PK_EPI_BF16 = 0,    /* out(bf16)[m,n] = alpha*acc + bias[n]                                     */
  PK_EPI_F32 = 1,     /* out(f32)[m,n]  = alpha*acc + bias[n] (+ out[m,n] when accumulate != 0)    */
  PK_EPI_GELU = 2,    /* out(bf16) = z = acc + bias ; out2(bf16) = gelu_erf(bf16(z))  (Mlp fc1+act) */
  PK_EPI_RESID = 3,   /* out(f32) = aux_f32[m,n] + rowscale[m / rows_per_group] * (acc + bias[n])
                         (residual add + DropPath scale, models_painter.py:229-230)               */
  PK_EPI_DGELU = 4,   /* out(bf16) = acc * gelu'(aux_bf16[m,n])        (backward through GELU)     */
  PK_EPI_PIXSHUF = 5, /* out(bf16) NHWC [B, h*p, w*p, c]: decoder_embed + 'nhwpqc->nchpwq' pixel
                         shuffle (models_painter.py:423-428), rows m=(b,i,j), cols n=(r,s,c)       */
};
typedef struct {
  int kind;
  void* out;
  void* out2;
  const float* bias;
  const void* aux;
  const float* rowscale;
  int ldc;            /* row stride of out/out2 (elements) */
  int ld_aux;         /* row stride of aux (elements) */
  int rows_per_group; /* rows sharing one rowscale entry */
  int accumulate;     /* PK_EPI_F32: 0 overwrite, 1 out += , 2 out zero-initialised, split-K atomics */
  float alpha;
  int ps_h, ps_w, ps_p, ps_c; /* pixel shuffle geometry: token grid h x w, patch p, channels c */
} PkEpilogue;

int pk_gemm_bf16(const void* A, const void* B, int M, int N, int K, int lda, int ldb, int transA,
                 int transB, const PkEpilogue* epi, void* stream);

/* test hooks: force the GEMM N-tile (64/128/256) or split-K factor; 0 restores the heuristics */
void pk_gemm_force_bn(int bn);
void pk_gemm_force_splits(int s);
/* Host-only views of the GEMM scheduler (schedule tests; no device work).  pk_gemm_plan: out9 = {cta_pair_kernel
 * (always 0: one CTA per 128 x BN tile), BN, row blocks, column blocks, splits, k-blocks per split, stream-K units per
 * CTA, raster group, workers}.
 * pk_gemm_plan_walk: the (row block, column block, kb0, kb1) items worker `worker` processes, 4 ints each; returns
 * minus the item count. */
int pk_gemm_plan(int M, int N, int K, int kind, int accumulate, int* out9);
int pk_gemm_plan_walk(int M, int N, int K, int kind, int accumulate, int worker, int* out4, int max_items);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm over channels (nn.LayerNorm(eps=1e-6): models_painter.py:193,200 norm1/norm2, :315,:417 final norm).
 * x fp32 [M, C] (row stride ldx) -> out (bf16 if out_is_bf16 else fp32; row stride ldo, so it can be a column
 * slice of the [M, 4C] decoder input, models_painter.py:422); mean/rstd [M] saved for backward (nullable).
 * bwd: dx = LN'(dy) (+ dres); dgamma/dbeta += column sums (caller initialises; deterministic two-stage
 * reduction through `workspace`).  dgamma = dbeta = NULL (frozen affine parameters): no reduction, `workspace`
 * may be NULL, dx is bit-identical.  In the _cast form each of dgamma, dbeta and colsum may be NULL on its own (that
 * sum is skipped; with all three NULL `workspace` may be NULL); dx and dx_bf16 are bit-identical.             */
int pk_layernorm_fwd(const float* x, int ldx, const float* gamma, const float* beta, float eps, void* out,
                     int ldo, int out_is_bf16, float* mean, float* rstd, int M, int C, void* stream);
long long pk_layernorm_bwd_ws_floats(int M, int C); /* fp32 elements of `workspace` (per-block partial sums) */
/* pk_layernorm_bwd fused with pk_scale_cast_colsum of its result (the backward of `x + drop_path(attn(norm1(x)))`
 * feeds norm2's input gradient, DropPath-scaled and cast to bf16, straight into the proj GEMMs; models_painter.py:
 * 216-235): also writes dx_bf16 = bf16(rowscale[row / rows_per_group] * dx) and adds its column sums to colsum[C]. */
int pk_layernorm_bwd_cast(const void* dy, int dy_is_bf16, int lddy, const float* x, int ldx, const float* mean, const float* rstd,
                          const float* gamma, const float* dres, float* dx, float* dgamma, float* dbeta,
                          float* workspace, const float* rowscale, int rows_per_group, void* dx_bf16, float* colsum,
                          int M, int C, void* stream);
int pk_layernorm_bwd(const void* dy, int dy_is_bf16, int lddy, const float* x, int ldx, const float* mean, const float* rstd,
                     const float* gamma, const float* dres, float* dx, float* dgamma, float* dbeta,
                     float* workspace, int M, int C, void* stream);

/* PatchEmbed lowering (util/vitdet_utils.py:178-186, models_painter.py:387-388): rows of (c,r,s)-ordered
 * patches of imgs then tgts, bf16 [2*B*h*w, Cin*p*p]; the conv itself is pk_gemm_bf16 on these rows.       */
int pk_im2col_patch(const float* imgs, const float* tgts, void* out_bf16, int B, int Cin, int H, int W, int p,
                    void* stream);
/* Input gradient of the PatchEmbed (prompt tuning, saliency): the exact inverse of pk_im2col_patch's layout.
 * dcols_x / dcols_y fp32 [B*h*w, Cin*p*p] (the patch-embed dgrad dE . W of the x rows / of the y rows; they may be the
 * two halves of one [2*B*h*w, Cin*p*p] buffer) -> dimgs / dtgts fp32 NCHW [B, Cin, H, W], overwritten.  Either output
 * may be NULL: its half of the columns is then not read and may be NULL too.                                  */
int pk_col2im_patch(const float* dcols_x, const float* dcols_y, float* dimgs, float* dtgts, int B, int Cin, int H,
                    int W, int p, void* stream);

/* Token assembly (models_painter.py:392-409; SegGPT type tokens models_seggpt.py:414-420) and its backward.
 * E fp32 [2B*N, C] (x rows then y rows); mask uint8 [maskB, N] (maskB = 1 broadcasts); pos fp32 [N, C];
 * type_emb fp32 [B, C] or NULL.  bwd: dE bf16 (y rows gated by 1-mask), dpos [N,C], dseg/dmask_token [C]
 * (atomically accumulated, caller zero-initialises).  Frozen parameters: dpos = NULL skips the position gradient,
 * dseg_x = dseg_y = dmask_token = NULL (all three) skips the token reductions; dE is unchanged.                 */
int pk_assemble_tokens(const float* E, const uint8_t* mask, int maskB, const float* mask_token,
                       const float* seg_x, const float* seg_y, const float* pos, const float* type_emb,
                       float* out, int B, int N, int C, void* stream);
int pk_assemble_tokens_bwd(const float* dZ, const uint8_t* mask, int maskB, void* dE_bf16, float* dpos,
                           float* dseg_x, float* dseg_y, float* dmask_token, int B, int N, int C, void* stream);
/* The same backward with the SegGPT type-token gradients (models_seggpt.py:415-420): seg_type fp32 [B] on the device;
 * dtype_cls / dtype_ins [C] (atomically accumulated, caller zero-initialises) receive sum_n (dZ[b, n] + dZ[B + b, n])
 * over the samples with seg_type[b] == 0 / == 1; other values contribute to neither.  dtype_cls = dtype_ins = NULL
 * (both) skips that reduction and seg_type is then not read.  pk_assemble_tokens_bwd is this call with all three
 * NULL; dE, dpos and the other token gradients do not depend on them.                                           */
int pk_assemble_tokens_bwd_typed(const float* dZ, const uint8_t* mask, int maskB, void* dE_bf16, float* dpos,
                                 float* dseg_x, float* dseg_y, float* dmask_token, const float* seg_type,
                                 float* dtype_cls, float* dtype_ins, int B, int N, int C, void* stream);

/* get_abs_pos (util/vitdet_utils.py:141-157): F.interpolate(bicubic, align_corners=False), NHWC [sh,sw,C] ->
 * [h,w,C]; bwd scatters atomically into a zero-initialised [sh,sw,C].                                      */
int pk_bicubic_fwd(const float* src, float* dst, int sh, int sw, int h, int w, int C, void* stream);
int pk_bicubic_bwd(const float* ddst, float* dsrc_accum, int sh, int sw, int h, int w, int C, void* stream);

/* Early merge (models_painter.py:414-415): out = 0.5*(z[:half] + z[half:]); bwd duplicates 0.5*d.          */
int pk_merge_halves(const float* z, float* out, long long half_elems, void* stream);
int pk_merge_halves_bwd(const float* d, float* out, long long half_elems, void* stream);

/* fp32 -> bf16 operand casts; optional per-row-group scale (DropPath backward, timm drop_path) and fused
 * column sums (bias gradients).                                                                           */
int pk_cast_bf16(const float* in, void* out_bf16, long long n, void* stream);
int pk_scale_cast_colsum(const float* in, int ldin, const float* rowscale, int rows_per_group, void* out_bf16,
                         float* colsum, int M, int C, void* stream);
int pk_colsum_bf16(const void* in_bf16, int ldin, float* colsum, int M, int C, void* stream);

/* Window attention plumbing (util/vitdet_utils.py:16-60 window_partition / window_unpartition; reachable only
 * through Painter(window_block_indexes=[...]), models_painter.py:220-227): zero-padded bf16 partition of the
 * [B,H,W,C] token grid into [B*nWh*nWw, ws, ws, C]; inverse: out = (resid or 0) + rowscale[b] * window value.   */
int pk_window_partition_bf16(const void* in, void* out, int B, int H, int W, int C, int ws, void* stream);
int pk_window_unpartition(const float* win, const float* resid, const float* rowscale, float* out, int B, int H,
                          int W, int C, int ws, void* stream);

/* SegGPT multi-prompt feature ensemble + residual (models_seggpt.py:220-231,:233): a, z, out fp32 [G*P, N, C]. */
int pk_ensemble_resid(const float* a, const float* z, float* out, int G, int P, int N, int C, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused attention with decomposed relative-position bias (models_painter.py:73-86 + util/vitdet_utils.py:
 * 63-125).  qkv bf16 [B*h*w, 3*heads*64] with columns (3, head, 64); th/tw = pk_relpos_table_bf16 outputs
 * (bf16, zero-padded to th_pad/tw_pad rows, multiples of 16); w must divide 112 (2,4,7,8,14,28,56).
 * fwd: out bf16 [B*N, heads*64], lse fp32 [B*heads, N] (log2 domain, nullable).
 * bwd: dqkv bf16 like qkv; dTh [2h-1,64], dTw [2w-1,64] fp32, added to (zero-initialise); dTh = dTw = NULL (frozen
 *      tables): no table gradients - the dQ kernel leaves out its G^T Q partials, the reduction kernel does not run,
 *      dt_ws may be NULL - and dqkv is bit-identical;
 *      scratch: delta [B*heads*N], relh_g [B*heads*Np*h], relw_g [B*heads*Np*w] (Np = N rounded up to 128), dt_ws
 *      [pk_attn_bwd_ws_floats(B, heads, h, w)] fp32 (per-CTA partial table gradients, reduced by a
 *      second kernel instead of same-address atomics).                                                     */
int pk_relpos_table_bf16(const float* table, void* out_bf16, int L, int Lpad, void* stream);
int pk_attn_fwd(const void* qkv, const void* th, const void* tw, void* out, float* lse, int B, int heads, int h,
                int w, int th_pad, int tw_pad, void* stream);
int pk_attn_bwd(const void* qkv, const void* O, const void* dO, const float* lse, const void* th, const void* tw,
                void* dqkv, float* dTh, float* dTw, float* delta, float* relh_g, float* relw_g, float* dt_ws,
                int B, int heads, int h, int w, int th_pad, int tw_pad, void* stream);
long long pk_attn_bwd_ws_floats(int B, int heads, int h, int w);
/* Training pair: pk_attn_fwd_save additionally stores every query's log2e-scaled bias rows (rel_h / rel_w of
 * vitdet_utils.py:113-123) in relh_g / relw_g (B*heads*Np*h resp. B*heads*Np*w floats, Np = N rounded up to 128; per
 * 128-query tile, query row innermost); pk_attn_bwd_saved takes them as INPUTS, so its dQ kernel starts from coalesced
 * loads instead of recomputing the two bias GEMMs and Toeplitz gathers.  Results are identical to pk_attn_fwd /
 * pk_attn_bwd.                                                                                                  */
int pk_attn_fwd_save(const void* qkv, const void* th, const void* tw, void* out, float* lse, float* relh_g,
                     float* relw_g, int B, int heads, int h, int w, int th_pad, int tw_pad, void* stream);
int pk_attn_bwd_saved(const void* qkv, const void* O, const void* dO, const float* lse, const void* th, const void* tw,
                      void* dqkv, float* dTh, float* dTw, float* delta, const float* relh_g, const float* relw_g,
                      float* dt_ws, int B, int heads, int h, int w, int th_pad, int tw_pad, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Decoder head (models_painter.py:328-333,430 decoder_pred = conv3x3 -> LayerNorm2D -> GELU -> conv1x1;
 * util/vitdet_utils.py:189-209) fused with forward_loss (:433-462) and patchify (:355-368).
 * g_nhwc: bf16 [B, H, W, 64] (output of the PK_EPI_PIXSHUF GEMM). wmat/wmat_t: pk_conv3x3_pack outputs.
 * head_params: fp32 [387] = conv3x3 bias[64] | LN2D weight[64] | LN2D bias[64] | conv1x1 weight[3][64] | bias[3].
 * fwd writes c1 (bf16 conv output, NHWC), patch_out fp32 [B, N, p*p*3] (= patchify(pred)), num[B] += sum
 * loss*mask*valid.  loss_kind: 0 smoothl1(beta .01), 1 l1, 2 l2, 3 l1l2.
 * pk_loss_prep: stats[b] = {sum (tgt*std+mean)*(1-M), sum M*valid};  pk_loss_finalize: loss + per-sample
 * coefficient keep_b/den (the `inds_ign` rule of :446-448; seggpt != 0 selects models_seggpt.py:457-468).      */
int pk_conv3x3_pack(const float* w, void* wf_bf16, void* wd_bf16, void* stream);
int pk_loss_prep(const float* tgts, const uint8_t* mask, int maskB, const float* valid, float* stats_zeroed,
                 int B, int H, int W, int p, void* stream);
int pk_decoder_head_fwd(const void* g_nhwc, const void* wmat, const float* head_params, const float* tgts,
                        const uint8_t* mask, int maskB, const float* valid, void* c1_out, float* patch_out,
                        float* num, int B, int H, int W, int p, int loss_kind, void* stream);
int pk_loss_finalize(const float* stats, const float* num, float* loss, float* coef, int B, int seggpt,
                     void* stream);
/* pk_decoder_head_bwd: dc1 (bf16 NHWC) and, when dhead_params_zeroed != NULL, the head parameters' gradients added
 * at offsets 64..386 of it (NULL: frozen head, no reductions; dc1 is bit-identical).
 * pk_decoder_head_bwd_dtgt: the same kernel, which also stores the loss's gradient with respect to the targets,
 * dtgts fp32 NCHW [B, 3, H, W] = -dpred = -(gscale * coef[b] * M * valid * dl/dd), d = pred - tgt (exact for
 * every loss_kind); it does not include the targets' path through the encoder.                               */
int pk_decoder_head_bwd(const void* c1, const float* tgts, const uint8_t* mask, int maskB, const float* valid,
                        const float* coef, const float* gscale, const float* head_params, void* dc1,
                        float* dhead_params_zeroed, int B, int H, int W, int p, int loss_kind, void* stream);
int pk_decoder_head_bwd_dtgt(const void* c1, const float* tgts, const uint8_t* mask, int maskB, const float* valid,
                             const float* coef, const float* gscale, const float* head_params, void* dc1,
                             float* dhead_params_zeroed, float* dtgts, int B, int H, int W, int p, int loss_kind,
                             void* stream);
int pk_conv3x3_dgrad_unshuffle(const void* dc1_nhwc, const void* wmat_t, void* out_tok, int B, int H, int W,
                               int p, void* stream);
int pk_conv3x3_wgrad(const void* g_nhwc, const void* dc1_nhwc, float* out, int B, int H, int W, void* stream);
int pk_conv3x3_wgrad_unpack(const float* acc, float* dw, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimizer step (SURVEY §8 f.1): fused multi-tensor AdamW with per-tensor lr / weight decay (the groups of
 * Painter/util/lr_decay.py:param_groups_lrd, main_train.py:344-348) and the global gradient norm of
 * util/misc.py:252-278.  `tensors_dev`: device array of PkOptTensor; `chunks_dev`: device array of int pairs
 * (tensor index, chunk index) - one CUDA block per chunk of pk_opt_chunk_elems() elements.  gscale (nullable device
 * scalar) multiplies every gradient (1 / loss scale, clip coefficient); gscale_cap > 0 clamps it from above
 * (clip coefficient min(1, .)).  pk_grad_sumsq adds sum(g^2) over all tensors to out_zeroed[0].
 * pk_droppath_scales: timm DropPath (0.3.2 layers/drop.py; models_painter.py:199,229-230) for a whole step in one
 * launch: out[i] = floor(round_to_dtype(keep[i] + r[i])) / keep[i], r = the torch.rand draws (dtype code 0 fp32,
 * 1 bf16, 2 fp16: the reference adds in the branch output's dtype).                                             */
typedef struct PkOptTensor {
  float* p;
  float* g;
  float* m;
  float* v;
  void* w16;      /* optional bf16 copy of p refreshed by the step (the tensor-core operand), or NULL */
  long long n;
  float lr, wd;
} PkOptTensor;
int pk_opt_chunk_elems(void);
/* zero_grad != 0: every gradient element is overwritten with 0 after it has been consumed (the flat gradient
 * arena is left clean for the next backward); found_inf (nullable device scalar): non-zero => the whole step is a
 * no-op (torch.cuda.amp.GradScaler.step semantics, util/misc.py:266). */
int pk_adamw_step(const PkOptTensor* tensors_dev, const int* chunks_dev, int nchunks, double beta1, double beta2,
                  double eps, int step, const float* gscale, float gscale_cap, int zero_grad,
                  const float* found_inf, void* stream);
/* pk_adamw_step for a CUDA-graph-captured training step (painter_b200.train_utils.GraphedTrainStep): the bias
   corrections 1 / (1 - beta1^t), 1 / sqrt(1 - beta2^t) are read from bc_dev[0..1] at run time. */
int pk_adamw_step_graph(const PkOptTensor* tensors_dev, const int* chunks_dev, int nchunks, double beta1,
                        double beta2, double eps, const float* bc_dev, const float* gscale, float gscale_cap,
                        int zero_grad, const float* found_inf, void* stream);
int pk_grad_sumsq(const PkOptTensor* tensors_dev, const int* chunks_dev, int nchunks, float* out_zeroed, void* stream);
int pk_droppath_scales(const void* r, int dtype_code, const float* keep, float* out, int n, void* stream);
/* Persistent kernels (the GEMM) use at most `n` SMs (0 = all): leaves room for a concurrent NCCL kernel
 * so that statically partitioned tiles never run as a second wave (multi-GPU backward).  Returns the old value. */
int pk_set_sm_budget(int n);
/* Programmatic dependent launch of the library's hot kernels (default on; PK_PDL=0 in the environment or
   pk_set_pdl(0) turns the launch attribute off).  Returns the previous setting. */
int pk_set_pdl(int on);

/* ------------------------------------------------------------------------------------------------
 * Inference pre/post-processing on the device (SURVEY §8 f.2).  Replaces the numpy / torch-CPU arithmetic around the
 * forward in SegGPT/SegGPT_inference/seggpt_engine.py:26-53 (run_one_image), :56-103 (inference_image), :106-181
 * (inference_video) and the run_one_image of the Painter eval scripts Painter/eval/ade20k_semantic/
 * painter_inference_segm.py:67-93, coco_panoptic/painter_inference_pano_{semseg,inst}.py, mmpose_custom/
 * painter_inference_pose.py, nyuv2_depth/painter_inference_depth.py and {sidd,lol,derain}/painter_inference_*.py.
 * dtype codes of image sources: 0 = uint8 (divided by 255.), 1 = fp32 in [0,1], 2 = fp64 in [0,1].
 *  pk_stitch_normalize  canvas[p,c,y,x] fp32 NCHW [P,3,2S,S] = ((top|bottom)[p][y%S,x,c] - mean_c) / std_c in fp64
 *                       (:75-91 stitch + ImageNet normalisation, :29-34 nhwc->nchw .float()); host arrays of P device
 *                       pointers
 *  pk_nhwc_to_nchw_f32  torch.einsum('nhwc->nchw', x).float() of an already normalised fp64/fp32 batch (:29-34)
 * pk_stitch_normalize takes any number of members (launched in chunks of 16).
 * De-normalisation and finishing, one launch for a whole batch (the per-image wrappers pass one image):
 *  pk_denorm_bottom_batched  out fp64 [B, h*p/2, w*p, 3] = finish(unpatchify(patch)[b * src_stride, bottom half]
 *                       * std + mean) (:48-52); finish: 0 = clip(x * 255, 0, 255), 1 = clip(x * 10000, 0, 10000)
 *                       (painter_inference_depth.py), 2 = x (painter_inference_{sidd,lol,derain}.py); bin (nullable,
 *                       finish 0 only) fp32 [B, h*p/2, w*p] = mean_c(out) > 128 (:164-169, video cache)
 *  pk_finish_ragged     one launch finishing n images of different output sizes from src fp64 [*, SH, SW, 3] with
 *                       `op` (PK_FIN_*).  items: int32 device table, one row of PK_RAG_FIELDS per image: [src sample,
 *                       OH, OW, cl_form, offset lo, hi]; the image's output starts at dst + offset (elements of the
 *                       op's output type: uint8, int32 for the depth, fp64 for the bicubic) and, for the blend, its
 *                       source image uint8 [OH, OW, 3] at image + offset (image is null for every other op).
 *                       max_pix >= every OH * OW sizes the grid.  The ops, as torch-CPU computes them on the float64
 *                       channels-last tensor:
 *     PK_FIN_BILINEAR_U8    dst uint8 [OH,OW,3] = uint8(int(bilinear(src))) (painter_inference_segm.py:89-92)
 *     PK_FIN_NEAREST_U8     dst uint8 [OH,OW,3] = uint8(int(nearest(src))) (painter_inference_pano_inst.py,
 *                           painter_inference_pose.py); cl_form selects torch-CPU's channels-last source index (it
 *                           takes that kernel when OH + OW <= 128), else its generic one
 *     PK_FIN_DEPTH          dst int32 [OH,OW] = int(bilinear(src).mean(-1)) (painter_inference_depth.py); cl_form
 *                           selects torch-CPU's channels-last summation order (it takes that kernel on one thread or
 *                           when OH + OW <= 128), else its generic one
 *     PK_FIN_BICUBIC_F64    dst fp64 [OH,OW,3] = F.interpolate(src, mode='bicubic'), unclipped
 *                           ({sidd,lol,derain} run_one_image, the returned array)
 *     PK_FIN_NEAREST_BLEND  dst uint8 [OH,OW,3] = uint8(image * (0.6 * nearest(src) / 255 + 0.4)) (:93-102)     */
enum { PK_RAG_FIELDS = 6 };
enum { PK_FIN_BILINEAR_U8 = 0, PK_FIN_NEAREST_U8 = 1, PK_FIN_DEPTH = 2, PK_FIN_BICUBIC_F64 = 3,
       PK_FIN_NEAREST_BLEND = 4 };
int pk_stitch_normalize(const void* const* top, const int* top_dtype, const void* const* bottom,
                        const int* bottom_dtype, float* out, int P, int S, void* stream);
int pk_nhwc_to_nchw_f32(const void* in, int in_is_f64, float* out, int n, int H, int W, void* stream);
int pk_denorm_bottom_batched(const float* patch, double* out, float* bin_or_null, int B, int src_stride, int h, int w,
                             int p, int finish, void* stream);
int pk_finish_ragged(int op, const double* src, int SH, int SW, const int* items, int n, int max_pix,
                     const uint8_t* image, void* dst, void* stream);

/* ------------------------------------------------------------------------------------------------
 * fp32-accurate forward mode (north star: within 1e-5 of the reference's fp32 forward, the way
 * seggpt_engine.run_one_image calls the model, seggpt_engine.py:47).  Every fp32 GEMM operand is split into three
 * bf16 terms (h, m, l) and the six significant cross products are evaluated by ONE pk_gemm_bf16 call over operands
 * concatenated along K: A' = [l|m|h|m|h|h], B' = [h|m|l|h|m|h] (K' = 6K, fp32 accumulation).
 *  pk_split3                 out bf16 [M, 6K] from x fp32 [M, K] (side_b: 0 = A-side, 1 = B-side order); gelu != 0
 *                            applies the exact erf GELU (timm Mlp act, models_painter.py:201) first
 *  pk_split3_heads           q / k / v of qkv fp32 [B*N, 3C] -> per-(b, head) operands of the attention GEMMs
 *                            (which: 0 q [B*heads, N, 384]; 1 k [B*heads, Npad, 384]; 2 v [B*heads, 6*Npad, 64])
 *  pk_softmax_relpos_split3  P' = split(softmax(scale * S + rel_h + rel_w)) (models_painter.py:80-86,
 *                            vitdet_utils.py:113-123) from S fp32 [BH, N, Npad], Gh = q.T_h^T, Gw = q.T_w^T
 *  pk_im2col_patch_split3    PatchEmbed im2col of imgs and tgts (vitdet_utils.py:178-186) as split A operand
 *  pk_dec_im2col_split3      pixel shuffle + 3x3 im2col of decoder_embed's output (models_painter.py:424-430)
 *  pk_head_f32               LayerNorm2D + exact GELU + conv1x1 + masked loss terms + patchify, fp32, from the fp32
 *                            conv3x3 output [B*H*W, 64]; num accumulates in fp64 (num_zeroed) and is emitted as fp32
 *  pk_attn_fwd_split3        fused attention with decomposed rel-pos bias in the same split arithmetic, without the
 *                            score matrix: qkv fp32 [B*h*w, 3C] (the qkv GEMM's layout), th / tw fp32 [2h-1, 64] /
 *                            [2w-1, 64] -> out fp32 [B*h*w, C] (heads merged).  h <= 112, w <= 56; a windowed block
 *                            calls it with B = all windows and h = w = window size.  No allocation or host sync.  */
int pk_split3(const float* x, int ldx, void* out_bf16, int M, int K, int side_b, int gelu, void* stream);
int pk_split3_heads(const float* qkv, void* out_bf16, int B, int heads, int N, int Npad, int which, void* stream);
int pk_softmax_relpos_split3(const float* S, const float* Gh, int ldgh, const float* Gw, int ldgw, void* P_bf16,
                             int BH, int N, int Npad, int h, int w, float scale, void* stream);
int pk_im2col_patch_split3(const float* imgs, const float* tgts, void* out_bf16, int B, int Cin, int H, int W, int p,
                           void* stream);
int pk_dec_im2col_split3(const float* D, void* out_bf16, int B, int h, int w, int p, int dd, void* stream);
int pk_head_f32(const float* c1, const float* head_params, const float* tgts, const uint8_t* mask, int maskB,
                const float* valid, float* patch, double* num_zeroed, float* num_out, int B, int H, int W, int p,
                int loss_kind, void* stream);
int pk_attn_fwd_split3(const float* qkv, const float* th, const float* tw, float* out, int B, int heads, int h, int w,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training data path, per-sample device work (SURVEY §8 f.4).
 *  pk_block_masks  BEiT block masks, one warp per sample: Painter/util/masking_generator.py:15-93 (blocks of random
 *                  area / log-uniform aspect ratio until num_masking cells are covered, then an exact-count fix-up) and
 *                  the half-mask alternative of Painter/data/pairdataset.py:149,183-186.  out int32 [B, H, W].
 *  pk_valid_maps   the per-task loss-weight maps of pairdataset.py:154-181.  rule[b]: 0 all ones; 1 valid[t < thr] = 0
 *                  (depth / semantic / panoptic-semantic); 2 valid[t > thr] = 10 and all 0 when fewer than 300
 *                  foreground values (pose); 3 all 0 when fewer than 300 foreground values (panoptic instances).
 *                  thr: fp32 [B, 3] normalised thresholds; fg_zeroed: int32 [B] scratch.                          */
int pk_block_masks(int* out, int B, int H, int W, int num_masking, int min_patches, int max_patches, float log_ar_lo,
                   float log_ar_hi, float half_mask_ratio, unsigned long long seed, void* stream);
int pk_valid_maps(const float* targets, const int* rule_dev, const float* thr_dev, int* fg_zeroed, float* valid, int B,
                  int H, int W, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training data path, the recipe's paired augmentations (Painter/main_train.py:232-262 as pairdataset.py applies them)
 * on decoded uint8 RGB images, bit-identical to PIL / torch-CPU given the host's random draws (csrc/augment.cu).
 * Descriptor tables are int32 device arrays, one row per job:
 *  crop row   [src byte offset lo, hi, H, W, top, left, h, w, mode (0 bicubic, 1 nearest), flip,
 *              tmp byte offset lo, hi]
 *  jitter row [slot, op0..op3 (PK_JIT_*, -1 = none, in the drawn order), brightness, contrast, saturation (float
 *              bits), hue shift (int(hue_factor * 255) mod 256)]
 *  second-crop row [top, left, h, w, mode (0 antialiased bicubic, 1 nearest)]; a full box in nearest mode is a copy.
 *  pk_aug_resized_crop  dst uint8 [J, S, S, 3] = resize(crop(src_j), S x S), flipped when asked (Pillow's resample).
 *                       KP >= every bicubic job's coefficient count (2 ceil(2 max(h, w) / S) + 1 bounds it);
 *                       max_rows >= every job's max(h, w); coef int32 [J, 2, S, KP], bounds int32 [J, 2, S, 2] and
 *                       tmp (the first pass, max(h, w) * S * 3 bytes per bicubic job at its offset) are scratch.
 *  pk_aug_color_jitter  ColorJitter (PIL) in place on images imgs + slot * npix * 3 (uint8 RGB), one CTA per image.
 *  pk_aug_normalize     ToTensor + Normalize + the two-pair stitch: slot (b * P + p) * 2 + t (t = 0 image, 1 target)
 *                       -> img / tgt fp32 [B, 3, P * S, S] rows p * S .. (p + 1) * S.
 *  pk_aug_second_crop   row 2b + t crops img / tgt [b] fp32 [3, OH, OW] and resizes it back to OH x OW
 *                       (torch-CPU interpolate, antialiased bicubic or nearest) into img_out / tgt_out.  wts fp32
 *                       [2B, 2, OH, PK_AUG_AA_TAPS], bounds int32 [2B, 2, OH, 2], tmp fp32 [2B, 3, OH, OW] scratch. */
enum { PK_AUG_CROP_FIELDS = 12, PK_AUG_JIT_FIELDS = 9, PK_AUG_SEC_FIELDS = 5, PK_AUG_AA_TAPS = 5 };
enum { PK_JIT_BRIGHTNESS = 0, PK_JIT_CONTRAST = 1, PK_JIT_SATURATION = 2, PK_JIT_HUE = 3 };
int pk_aug_resized_crop(const uint8_t* src, const int* jobs, int J, int S, int KP, int max_rows, int* coef, int* bounds,
                        uint8_t* tmp, uint8_t* dst, void* stream);
int pk_aug_color_jitter(uint8_t* imgs, const int* jobs, int n, long long npix, void* stream);
int pk_aug_normalize(const uint8_t* slots, int B, int P, int S, float* img, float* tgt, void* stream);
int pk_aug_second_crop(const float* img, const float* tgt, const int* jobs, int B, int OH, int OW, float* wts,
                       int* bounds, float* tmp, float* img_out, float* tgt_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Task metrics (csrc/metrics.cu, painter_b200/task_metrics.py): the scores of the reference's evaluators from the eval
 * outputs on the device, with no host round trip.  A launch covers a batch of images described by an int64 device
 * table, one row of PK_METRIC_FIELDS per image: [pred, pred_staged, gt offset, H, W].  pred is the prediction's device
 * address, or its byte offset from `base` when pred_staged != 0; the ground truth is at base + gt offset (base: the
 * caller's upload buffer).
 *  pk_palette_classes     out uint8 [npix] = argmin_k dist(segm[i], palette[k]), the first minimum, with the distance of
 *                         SemSegEvaluatorCustom.post_process_segm_output (Painter/eval/ade20k_semantic/
 *                         ADE20kSemSegEvaluatorCustom.py:114-141): PK_DIST_ABS sum |c - P|, PK_DIST_SQUARE sum (c - P)^2,
 *                         PK_DIST_MEAN sum (|c - P| + (c - P)^2) / 2.  segm uint8 [npix, 3], palette uint8 [K, 3],
 *                         1 <= K <= 200.
 *  pk_semseg_confusion    conf int64 [(K+1) * (K+1)] += the counts of cell (K + 1) * class(pred) + gt over every pixel
 *                         of the n images (pred uint8 [H, W, 3], gt uint8 [H, W]; gt == ignore_label counts as K), as
 *                         the evaluator's np.bincount (:96-101).  Labels >= K other than ignore_label are the caller's
 *                         to refuse.  max_pix >= every H * W sizes the grid.
 *  pk_depth_errors        out fp64 [n, 9] = {d1, d2, d3, AbsRel, SqRel, RMSE, RMSElog, SILog, log10} of Painter/eval/
 *                         nyuv2_depth/eval_with_pngs.py (pred int32 [H, W] / 1000 clamped into [min_depth, max_depth],
 *                         gt uint16 [H, W] / 1000, pixels min_depth < gt < max_depth, Eigen crop rows 45:471, columns
 *                         41:601 when eigen_crop != 0).  One CTA per image.
 *  pk_restoration_scores  psnr, ssim fp64 [n]: skimage 0.19 peak_signal_noise_ratio(x, y) and structural_similarity(
 *                         x, y, multichannel=True) as Painter/eval/lol/painter_inference_lol.py calls them, x =
 *                         clip(pred, 0, 1) (pred fp64 [H, W, 3]), y = gt / 255. (gt uint8 [H, W, 3]); c1, c2 the SSIM
 *                         constants.  Every image is at least 7 x 7; max_h, max_w bound every H, W.  counters_zeroed
 *                         uint32 [n] (zero on entry); partials fp64 [n * pk_restoration_ws_doubles(max_h, max_w)].
 * All results are bitwise reproducible (integer sums, or fp64 sums in a fixed order).                             */
enum { PK_METRIC_FIELDS = 5 };
enum { PK_DIST_ABS = 0, PK_DIST_SQUARE = 1, PK_DIST_MEAN = 2 };
int pk_palette_classes(const uint8_t* segm, long long npix, const uint8_t* palette, int K, int dist_type, uint8_t* out,
                       void* stream);
int pk_semseg_confusion(const long long* items, const void* base, int n, long long max_pix, const uint8_t* palette,
                        int K, int dist_type, int ignore_label, long long* conf, void* stream);
int pk_depth_errors(const long long* items, const void* base, int n, float min_depth, float max_depth, int eigen_crop,
                    double* out, void* stream);
long long pk_restoration_ws_doubles(int max_h, int max_w);
int pk_restoration_scores(const long long* items, const void* base, int n, int max_h, int max_w,
                          unsigned* counters_zeroed, double* partials, double c1, double c2, double* psnr, double* ssim,
                          void* stream);

/* ------------------------------------------------------------------------------------------------
 * MATLAB-scored restoration benchmarks (csrc/restoration_matlab.cu, painter_b200/task_metrics.py derain_scores,
 * sidd_scores, ycbcr_y), restated from the scripts and MATLAB's documented algorithms (unverified against MATLAB).
 * Same descriptor table as the task metrics above: pred fp64 [H, W, 3], gt uint8 [H, W, 3].
 *  pk_ycbcr_y          out uint8 [npix] = the Y channel of MATLAB rgb2ycbcr of rgb uint8 [npix, 3]: K1 R + K2 G + K3 B
 *                      + 16 in fp64 with Ki = (1/255) * {65.481, 128.553, 24.966}, summed left to right without FMA,
 *                      rounded half away from zero, saturated.
 *  pk_derain_scores    psnr, ssim fp64 [n]: Painter/eval/derain/evaluate_PSNR_SSIM.m compute_psnr and SSIM_index on the
 *                      Y channels of u = uint8(trunc(clip(pred, 0, 1) * 255)) and gt; C1 = (0.01 * 255)^2, C2 =
 *                      (0.03 * 255)^2 as c1, c2; taps fp64 [11] the normalised 1-D Gaussian (sigma 1.5) whose outer
 *                      product is the SSIM window.  Every image is at least 11 x 11.
 *  pk_sidd_scores      psnr, ssim fp64 [n]: MATLAB psnr and ssim as Painter/eval/sidd/eval_sidd.m calls them, x =
 *                      single(clip(pred, 0, 1)), y = single(gt) / 255 (H x W x 3 volume, replicate padding); consts fp64
 *                      [20]: the 11 taps, then the 3 x 3 depth-filter matrix row by row; c1 = 0.01^2, c2 = 0.03^2.
 *  Both: max_h, max_w bound every H, W; counters_zeroed uint32 [n] (zero on entry); partials fp64
 *  [n * pk_{derain,sidd}_ws_doubles(max_h, max_w)].  One CTA per (16 x 16 tile, image); bitwise reproducible.    */
int pk_ycbcr_y(const uint8_t* rgb, long long npix, uint8_t* out, void* stream);
long long pk_derain_ws_doubles(int max_h, int max_w);
long long pk_sidd_ws_doubles(int max_h, int max_w);
int pk_derain_scores(const long long* items, const void* base, int n, int max_h, int max_w, const double* taps,
                     unsigned* counters_zeroed, double* partials, double c1, double c2, double* psnr, double* ssim,
                     void* stream);
int pk_sidd_scores(const long long* items, const void* base, int n, int max_h, int max_w, const double* consts,
                   unsigned* counters_zeroed, double* partials, double c1, double c2, double* psnr, double* ssim,
                   void* stream);

/* ------------------------------------------------------------------------------------------------
 * COCO panoptic post-processing (csrc/panoptic.cu, painter_b200/panoptic.py): Painter/eval/coco_panoptic's instance
 * decoding, matrix NMS, class vote and panoptic merge on the device.  A launch covers a batch of n images described by
 * an int64 device table, one row of PK_PANO_FIELDS per image: [pixels, staged, H, W].  pixels is the uint8 [H, W, 3]
 * image's device address, or its byte offset from `base` when staged == 1.  Mask tables (pack_masks, unpack outputs)
 * hold [bool / int32 [.., H, W] device address, rows, H, W].  Per image, `ncap` rows of `words` uint32 (a multiple of
 * 32) hold the bit rows of its masks (bit p of row i: pixel p in mask i).
 *  pk_pano_candidates     area int32 [n, T, P], sumfx int64 [n, T, P] (zeroed by the caller) += the pixel count and the
 *                         2^-25 fixed-point sum of dist = fp32(L1) * fp32(1/3) of candidate (t, c) = {p : L1(p, P_c) <
 *                         bounds[t]} (COCOCAInstSegEvaluatorCustom.py:283-299, the (num_color, h, w) dist / mask
 *                         tensors); P <= PK_PANO_MAX_PALETTE colours, T <= PK_PANO_MAX_THR thresholds.
 *  pk_pano_select         the non-empty candidates sorted stably by (maskness, t * P + c), the first `keep`: count
 *                         int32 [n], cand int32 [n, ncap], scores fp32 [n, ncap] = 1 - m / max(max m, 1) (:312-325).
 *                         ws: pk_pano_select_ws_bytes(n, T * P) bytes.
 *  pk_pano_pack_candidates  bits of the kept candidates cand[i], i < count.
 *  pk_pano_pack_masks     bits of explicit bool masks (one table row per image); aux int64 [n, 2] rows [fp32 scores
 *                         address, int64 classes address or 0] gathered into scores fp32 / classes int64 [n, ncap].
 *  pk_pano_gram           gram int32 [n, ncap, ncap]: popc(row_i & row_j) on every 128 x 128 tile on or above the
 *                         diagonal with a row below count (util/matrix_nms.py:64-67 inter_matrix); ncap a multiple
 *                         of 128.
 *  pk_pano_nms            mask_matrix_nms (util/matrix_nms.py:53-121, gaussian kernel, filter_thr -1, nms_pre -1):
 *                         rows int32 [n, max_num] (input indices), out_scores fp32 [n, max_num], out_count [n],
 *                         out_labels int64 [n, max_num] or null (labels[row], 1 without labels).  labels
 *                         int64 [n, ncap] or null (class-agnostic); gram null: no decay, the stable descending order
 *                         only.  empty_one: an image without candidates gets one row -1 with score 0 (:301-310).
 *                         ws: 4 * n * ncap int32.
 *  pk_pano_unpack         bool masks out[i] = row rows[img * rows_ld + i] (zeros for -1).
 *  pk_pano_minmax         post_process_segm_output_by_minmax (:172-250): pred int16 [n, max_pix] = the first nearest
 *                         of the P colours and black (index P); cnt, sum [n, P + 1] (zeroed); cols / scores / classes
 *                         [n, P + 1] and count [n]: the colours present in index order.
 *  pk_pano_minmax_masks   bool masks out[i] = (pred == cols[img * P1 + i]).
 *  pk_pano_vote           classes int64 [n, ncap] = argmax_k sum over the mask of 1 - d_k / max d (k < 80, d the L1
 *                         distance to semantic colour k; COCOPanoEvaluatorCustom.py:259-276); dmax_zeroed int32 [n].
 *  pk_pano_merge          combine_semantic_and_instance_outputs_custom (COCOPanoEvaluatorCustom.py:47-134): int32
 *                         maps (zeroed) from the instances' bits / scores / classes and the semantic argmin map (labels
 *                         uint8 [n, max_pix] workspace; 80 <= K <= 200); segs int64 [n, max_seg, 4] = {instance or -1,
 *                         category, area, fp32 score bits}, nseg int32 [n].
 * All results are bitwise reproducible (integer sums and counts, stable orders on explicit keys).                  */
enum { PK_PANO_FIELDS = 4, PK_PANO_MAX_PALETTE = 6400, PK_PANO_MAX_THR = 4 };
int pk_pano_candidates(const long long* items, const void* base, int n, long long max_pix, const uint8_t* palette,
                       int P, const int* bounds, int T, int* area, long long* sumfx, void* stream);
long long pk_pano_select_ws_bytes(int n, int NC);
int pk_pano_select(const int* area, const long long* sumfx, int n, int NC, int keep, int ncap, void* ws,
                   long long ws_bytes, int* count, int* cand, float* scores, void* stream);
int pk_pano_pack_candidates(const long long* items, const void* base, int n, const uint8_t* palette, int P,
                            const int* bounds, int T, const int* cand, const int* count, int ncap, int words,
                            uint32_t* bits, void* stream);
int pk_pano_pack_masks(const long long* items, int n, int max_rows, int ncap, int words, uint32_t* bits,
                       const long long* aux, float* scores, long long* classes, void* stream);
int pk_pano_gram(const uint32_t* bits, int n, int ncap, int words, const int* count, int* gram, void* stream);
int pk_pano_nms(const int* gram, const long long* labels, const float* scores, const int* count, int n, int ncap,
                float sigma, int max_num, int empty_one, int* ws, int* rows, float* out_scores, int* out_count,
                long long* out_labels, void* stream);
int pk_pano_unpack(const uint32_t* bits, int n, int ncap, int words, const int* rows, int rows_ld, int max_rows,
                   long long max_pix, const long long* outs, void* stream);
int pk_pano_minmax(const long long* items, const void* base, int n, long long max_pix, const uint8_t* palette, int P,
                   short* pred, int* cnt, long long* sum, int* cols, float* scores, long long* classes, int* count,
                   void* stream);
int pk_pano_minmax_masks(const short* pred, int n, long long max_pix, const int* cols, int P1, int max_rows,
                         const long long* outs, void* stream);
int pk_pano_vote(const long long* items, const void* base, int n, long long max_pix, const uint8_t* palette,
                 const uint32_t* bits, int ncap, int words, const int* count, int max_rows, int* dmax_zeroed,
                 long long* classes, void* stream);
long long pk_pano_merge_smem(int words, int ncap);
int pk_pano_merge(const long long* sem_items, const void* base, const long long* maps, int n, long long max_pix,
                  const uint8_t* palette, int K, uint8_t* labels, const uint32_t* bits, int ncap, int words,
                  const float* scores, const long long* classes, const int* count, double overlap, double stuff_area,
                  double score_thresh, int max_seg, long long* segs, int* nseg, void* stream);

/* ------------------------------------------------------------------------------------------------
 * COCO pose post-processing (csrc/pose.cu, painter_b200/pose.py): Painter/eval/mmpose_custom's heatmap decoding, flip
 * averaging, keypoint decoding, rescoring and OKS NMS on the device.
 *  pk_pose_decode   out fp32 [n, 17, 3] = (x, y, maxval) of forward_pseudo_test + the head's decode (model/top_down.py
 *                   :163-258; flip_test iff flipped images are given, shift_heatmap, post_process 'default', no UDP).
 *                   items int64 [n, PK_POSE_FIELDS] rows [pred, pred staged, flipped, flipped staged]: a uint8
 *                   [H, W, 3] image's device address, or its byte offset from `base` when staged == 1; flipped staged
 *                   == 2: no flipped image (all rows alike).  palette: host uint8 [18, 2] (G, B); swap: host int32 [17]
 *                   (flip_back's channel swap); cs fp32 [n, 4] rows (center x, y, scale x, y); keys_zeroed u64
 *                   [n, 17] and done_zeroed u32 [n] zeroed workspace.  H, W >= 3.
 *  pk_pose_nms      the rescoring and oks_nms of data/topdown_coco_dataset.py:266-297 for n_img images, one CTA each:
 *                   images int32 [n_img, 2] rows (start, count) into pos int32 (box rows of kpts fp32 [N, 51],
 *                   box_scores fp32 [N], areas fp32 [N]), each image's boxes in bbox_id order, count <= 1024.  vars:
 *                   host fp64 [17] = (2 sigma)^2.  Order: score descending, ties the later box first.  rows int32
 *                   [sum count, PK_POSE_ROW] from each image's start, in keep order: (pos, fp32 score bits, 51 fp32
 *                   keypoint bits); counts int32 [n_img] kept.  Shared memory: pk_pose_nms_smem(max count).
 * Results are bitwise reproducible (key maxima, explicitly rounded arithmetic, explicit orders).                     */
enum { PK_POSE_FIELDS = 4, PK_POSE_JOINTS = 17, PK_POSE_PALETTE = 18, PK_POSE_MAX_BOXES = 1024, PK_POSE_ROW = 53 };
int pk_pose_decode(const long long* items, const void* base, int n, int H, int W, const uint8_t* palette,
                   const int* swap, const float* cs, unsigned long long* keys_zeroed, unsigned* done_zeroed,
                   float* out, void* stream);
long long pk_pose_nms_smem(int max_count);
int pk_pose_nms(const int* images, int n_img, int max_count, const int* pos, const float* kpts,
                const float* box_scores, const float* areas, const double* vars, float vis_thr, float oks_thr,
                int* rows, int* counts, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PAINTER_B200_H */

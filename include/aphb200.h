/* aphb200.h -- C ABI of libaphb200.so: the H100-native (sm_90a) hot path of eps696/aphantasia.
 *
 * Drop-in boundary (SURVEY.md section 8b). Plain pointers and sizes only; no torch types. Every compute entry
 * point is asynchronous on the caller's `stream` (pass torch.cuda.current_stream().cuda_stream as void*),
 * returns 0 on success / non-zero on error (message: aph_last_error(), thread-local), and never owns
 * user-visible memory: inputs/outputs are caller-owned DEVICE pointers (fp32 unless stated). Scratch lives
 * in library-owned handles so it survives the reference's per-step torch.cuda.empty_cache()
 * (/root/reference/clip_fft.py:285).
 *
 * Each entry point cites the reference interface it replaces (paths relative to /root/reference).
 * The Python binding (ctypes) is aphantasia_b200/_lib.py; INTEGRATION.md shows the reference-side stub.
 */
#ifndef APHB200_H_
#define APHB200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define APH_ABI_VERSION 1

/* ---- crop parameter table: one row per crop, APH_CROP_PARAM_FLOATS float32 values.
 * Built on the host by replaying the reference's RNG order (aphantasia_b200/_rng.py).               */
#define APH_CROP_PARAM_FLOATS 24
#define APH_F_OFFY   0   /* crop top-left y in the sampling frame (integer-valued)   utils.py:247 */
#define APH_F_OFFX   1   /* crop top-left x                                          utils.py:246 */
#define APH_F_CSIZE  2   /* crop side in canvas pixels                                utils.py:245 */
#define APH_F_FLAGS  3   /* bit0 perspective, bit1 erase, bit2 rotate, bit3 jitter, bit4 elastic    */
#define APH_F_PERSP  4   /* 8 coeffs a..h, output->input (torchvision _get_perspective_coeffs)     */
#define APH_F_ER_I   12  /* erase rect top, left, height, width (torchvision RandomErasing)        */
#define APH_F_ER_J   13
#define APH_F_ER_H   14
#define APH_F_ER_W   15
#define APH_F_ROT    16  /* theta00, theta01, theta10, theta11 of the inverse affine matrix. For APH_TF_CUSTOM /
                          * APH_TF_ELASTIC: the pixel-space inverse rotation of kornia's warp_affine about
                          * c = (s-1)/2, s = size + 8: source = c + [[r00, r01], [r10, r11]] (dest - c), (x, y) order */
#define APH_F_ANGLE  20  /* degrees, informational                                                 */
#define APH_F_JIT_DX 21  /* APH_TF_CUSTOM / APH_TF_ELASTIC: integer jitter shift (kornia translate): */
#define APH_F_JIT_DY 22  /*   out(x, y) = in(x - dx, y - dy), zero outside                          */
#define APH_FLAG_PERSP   1
#define APH_FLAG_ERASE   2   /* for APH_TF_ELASTIC the rectangle is in the padded (size + 8) image  */
#define APH_FLAG_ROT     4
#define APH_FLAG_JITTER  8
#define APH_FLAG_ELASTIC 16  /* kornia elastic_transform2d with zero noise: a 1-D bilinear stretch per axis */

/* sampler transform kinds (what `transform=` of slice_imgs was)                                  */
#define APH_TF_NONE      0   /* bicubic resize only                                                */
#define APH_TF_NORMALIZE 1   /* + transforms.normalize()            transforms.py:102-109          */
#define APH_TF_FAST      2   /* transforms.transforms_fast          transforms.py:165-170          */
/* The next two write [S,3,size+8,size+8]: pad(4, 0.5) -> [erase] -> rotate (bilinear, zeros) -> [elastic stretch]
 * -> jitter(8) -> normalise, each stage a resampling of the (size+8)^2 image.                                       */
#define APH_TF_CUSTOM    3   /* transforms.transforms_custom        transforms.py:156-163          */
#define APH_TF_ELASTIC   4   /* transforms.transforms_elastic       transforms.py:147-154          */

/* similarity kinds (sim_func `type`)                                         utils.py:276-295    */
#define APH_SIM_COS 0
#define APH_SIM_MIX 1

int         aph_version(void);
const char* aph_last_error(void);

/* ================= L3: spectrum -> RGB synthesis =============================================
 * Replaces fft_image.inner (aphantasia/image.py:164-175) and, fused, to_valid_rgb.inner
 * (aphantasia/image.py:21-28):   x = irfftn(scale*(P [+shift]), s=(H,W), 'ortho');
 *                                 img = x*contrast/std(x);  out = sigmoid(colmat . img)            */
typedef struct aph_fft_plan aph_fft_plan;
int aph_fft_plan_create(aph_fft_plan** plan, int H, int W);   /* H, W: prime factors <= 13 */
int aph_fft_plan_destroy(aph_fft_plan* plan);

/* params [3,H,Wh,2], scale [H,Wh] (Wh = W/2+1).  shift_mode 0: none; 1: shift [H,Wh] (the script's
 * --noise, clip_fft.py:238); 2: shift [3,H,Wh,2] (illustra.py:334).
 * colmat: 9 floats, HOST pointer, row-major Mn[d][c] (out_d = sum_c Mn[d][c] img_c) or NULL = no
 * decorrelation. apply_sigmoid 0/1.
 * Outputs: x_raw [3,H,W] (un-normalised irfft, saved for backward), stats double[4] on device
 * {sum x, sum x^2, sum g.x (bwd scratch), unused}, out [3,H,W].                                    */
int aph_synth_fft_fwd(aph_fft_plan* plan, const float* params, const float* scale,
                      const float* shift, int shift_mode, float contrast,
                      const float* colmat_host, int apply_sigmoid,
                      float* x_raw, double* stats, float* out, void* stream);
/* grad_out [3,H,W] = dL/d out  ->  grad_params [3,H,Wh,2] (overwritten).                           */
int aph_synth_fft_bwd(aph_fft_plan* plan, const float* grad_out, const float* out,
                      const float* x_raw, double* stats, const float* scale, float contrast,
                      const float* colmat_host, int apply_sigmoid,
                      float* grad_params, void* stream);

/* ---- starting from an image file (resume_fft / img2fft / img2dwt / pixel_image, aphantasia/image.py:82-107,130-150,185-220).
 * aph_un_rgb: un_rgb (image.py:185-197). hwc: DEVICE uint8 [H,W,3] (grey / RGBA are made 3-channel on the host, as
 * utils.img_read does); out [3,H,W] = gain * Minv . ((x/255 - mean) / std) with the CLIP normalisation of transforms.py:106;
 * inv_colmat_host: 9 floats, HOST, row-major Minv[d][c] = inverse(colcorr_t)[c][d] (the inverse of to_valid_rgb's mix).
 * gain is 1 (img2fft / img2dwt) or 3.3 (pixel_image).                                                               */
int aph_un_rgb(const uint8_t* hwc, int H, int W, const float* inv_colmat_host, float gain, float* out, void* stream);
/* aph_fft_analyze: spectrum [3,H,Wh,2] = ascale [H,Wh] * rfftn(img [3,H,W], norm='ortho') on a plan of the image's size.
 * img2fft's division by un_spectrum's scale, its factor 500000 and resume_fft's sd are all folded into ascale. Uses the
 * plan's scratch: do not interleave with a synthesis on the same plan and stream order.                              */
int aph_fft_analyze(aph_fft_plan* plan, const float* img, const float* ascale, float* spectrum, void* stream);

/* Wavelet parameterisation (BASELINE config 3). Replaces dwt_image.inner (aphantasia/image.py:66-69):
 *   img = DWTInverse((Yl, [Yh_i * scale_i])) * contrast / std, fused with to_valid_rgb like the FFT path.
 * DWTInverse is pytorch_wavelets' (third-party, mode 'symmetric'); rec_lo / rec_hi (HOST, L taps) are the
 * PyWavelets reconstruction filters. J = floor(log2(min(H, W))) levels (image.py:35-36).                        */
typedef struct aph_dwt_plan aph_dwt_plan;
int aph_dwt_plan_create(aph_dwt_plan** plan, int H, int W, const float* rec_lo_host, const float* rec_hi_host, int L);
int aph_dwt_plan_destroy(aph_dwt_plan* plan);
/* J; dims[2*i], dims[2*i+1] = band height/width of level i+1 (finest first); out_hw = synthesised image size      */
int aph_dwt_plan_levels(const aph_dwt_plan* plan, int* J, int* dims, int* out_hw);
/* Ys: HOST array of J+1 DEVICE pointers {Yl [3,hJ,wJ], Yh_1 [3,3,h1,w1] (finest), ..., Yh_J}; scales_host [J]
 * (aphantasia/image.py:73-80). Outputs as aph_synth_fft_fwd (x_raw / out are [3,out_h,out_w]).                    */
int aph_synth_dwt_fwd(aph_dwt_plan* plan, const float* const* Ys, const float* scales_host, float contrast,
                      const float* colmat_host, int apply_sigmoid, float* x_raw, double* stats, float* out,
                      void* stream);
/* grad_Ys: HOST array of J+1 DEVICE pointers receiving d loss / d Ys (overwritten).
 * Adam fused into the backward (the trailing arguments; params == NULL: none): params / m / v (and vmax, may be NULL) are
 * HOST arrays of J+1 DEVICE pointers ordered as Ys, every tensor updated in place by step `step` of aph_adam_step where
 * its gradient is formed. grad_Ys may then be NULL (nothing is written).                                               */
int aph_synth_dwt_bwd(aph_dwt_plan* plan, const float* grad_out, const float* out, const float* x_raw,
                      double* stats, const float* scales_host, float contrast, const float* colmat_host,
                      int apply_sigmoid, float* const* grad_Ys, void* stream,
                      float* const* params, float* const* m, float* const* v, float* const* vmax,
                      float lr, float b1, float b2, float eps, float weight_decay, int step);
/* Analysis of an image (img2dwt, aphantasia/image.py:82-94): DWTForward(J, wave, mode='symmetric') of img [3,H,W] (H, W of
 * the plan), rows filtered before columns, bands (LH, HL, HH). Ys: HOST array of J+1 DEVICE pointers shaped as for
 * aph_synth_dwt_fwd, overwritten; Yh_i is multiplied by inv_scales_host[i] (HOST [J]). Uses the plan's LL scratch; the
 * row-filtered halves of each level live in a stream-ordered allocation (cudaMallocAsync) freed behind that level.        */
int aph_dwt_analyze(aph_dwt_plan* plan, const float* img, const float* inv_scales_host, float* const* Ys, void* stream);

/* Direct RGB parameterisation: pixel_image.inner (aphantasia/image.py:112-118): img = x*contrast/std(x) (or /3.3 with
 * fixcontrast), fused with to_valid_rgb. x / out / grad_x are [3,H,W]; stats as above.                             */
int aph_pixel_fwd(const float* x, int64_t hw, float contrast, int fixcontrast, const float* colmat_host,
                  int apply_sigmoid, double* stats, float* out, void* stream);
/* Adam fused into the backward (the trailing arguments; params == NULL: none): params / m / v (and vmax, may be NULL)
 * [3,H,W] are updated in place by step `step` of aph_adam_step from d loss / d x; params may be x itself. grad_x is then
 * scratch, and does not receive the gradient.                                                                        */
int aph_pixel_bwd(const float* grad_out, const float* out, const float* x, double* stats, int64_t hw, float contrast,
                  int fixcontrast, const float* colmat_host, int apply_sigmoid, float* grad_x, void* stream,
                  float* params, float* m, float* v, float* vmax, float lr, float b1, float b2, float eps,
                  float weight_decay, int step);

/* Stand-alone to_valid_rgb for a foreign image_f (aphantasia/image.py:21-28): img [3,H,W] -> out.  */
int aph_valid_rgb_fwd(const float* img, int64_t hw, const float* colmat_host, float* out, void* stream);
int aph_valid_rgb_bwd(const float* grad_out, const float* out, int64_t hw, const float* colmat_host,
                      float* grad_img, void* stream);

/* ================= per-frame camera motion (illustrip.py) =====================================
 * Replaces frame_transform's T.functional.affine(img, angle, shift, scale, shear, fill=0, interpolation=BILINEAR)
 * (illustrip.py:130-138) on a CUDA tensor: torchvision's _gen_affine_grid (pixel-centre grid, align_corners=False),
 * grid_sample bilinear with zero padding, and the fill-0 blend out = sample(img) * sample(ones). Forward only.
 * in / out [planes,H,W] (must not alias); inv_matrix_host: 6 doubles, HOST, the inverse matrix of torchvision's
 * _get_inverse_affine_matrix (centre (0, 0) = the image centre). One launch.                                      */
int aph_affine_fwd(const float* in, int planes, int H, int W, const double* inv_matrix_host, float* out, void* stream);

/* ================= CPPN generator (cppn.py) ===================================================
 * Replaces CPPN.forward (cppn.py:71-116): a per-pixel MLP from the coordinate to RGB, written as 1x1 convolutions.
 * Layer 0: 2 -> nf; layers 1 .. layers-1: kh -> nf; output: kh -> 3, sigmoid. kh = 2 nf for act 0 `unbias`
 * (t = atan z, cat(t / 0.67, (t^2 - 0.45) / 0.396)) and act 1 `comp` (cat(t / 0.67, t^2 / 0.6)), kh = nf for act 2 `relu`
 * ((relu z - 0.4) / 0.58). The hidden layers' products run in TF32 (operands rounded by cvt.rna), everything else in fp32.
 * aph_cppn_create accepts nf a multiple of 8 in [8, 256] and layers in [1, 32] and refuses anything else (host only, no GPU
 * work). The handle owns the scratch of both calls. nf <= 64 keeps each pixel's activations in registers (no scratch for the
 * forward; the backward's per-CTA partials). 72 <= nf <= 256 runs layer by layer over all pixels, the hidden layers as TF32
 * wgmma GEMMs, and grows one buffer to 4 F bytes, for P = N H W pixels:
 *   chunk = max(4096, ceil(ceil(P / 256) / 128) * 128), S = ceil(P / chunk), Pp = S chunk, R = Pp / 16,
 *   KHP = KH rounded up to 128 (KH <= 128) or to 256, Q = 3 KH + 8 + nf,
 *   forward:  F = 2 Pp KH + (layers - 1) nf KH
 *   backward: F = 2 Pp KH + 2 (layers - 1) nf KH + layers nf Pp + KHP Pp + nf Pp + max(R Q, S nf KH) + 2 ceil(R / 256) Q
 * (512 x 512, nf 256, 10 layers: 1.1 GB forward, 4.7 GB backward). A failed allocation returns an error naming the size.
 * params / dparams: HOST arrays of 2 (layers + 1) DEVICE pointers {W0, b0, W1, b1, ..., W_layers, b_layers}, W_l the
 * nn.Conv2d weight [out, in, 1, 1] (8-byte aligned), read in place by every call.
 * coords [N,2,H,W] -> out [N,3,H,W]; pixel p = n H W + h W + w. One launch for nf <= 64, layers + 2 above.          */
typedef struct aph_cppn aph_cppn;
int aph_cppn_create(aph_cppn** handle, int nf, int layers, int act);
int aph_cppn_destroy(aph_cppn* handle);
/* device bytes the handle holds now (its scratch grows to the largest call so far)                                    */
int64_t aph_cppn_bytes(const aph_cppn* handle);
int aph_cppn_fwd(aph_cppn* handle, const float* coords, int N, int H, int W, const float* const* params, float* out,
                 void* stream);
/* grad_out [N,3,H,W] -> every dparams tensor (overwritten); no coordinate gradient. Recomputes the forward. Two launches
 * for nf <= 64, a few per layer above; the weight gradient is reduced in a fixed order, so repeated calls give bit-identical
 * results.                                                                                                              */
int aph_cppn_bwd(aph_cppn* handle, const float* coords, int N, int H, int W, const float* const* params,
                 const float* grad_out, float* const* dparams, void* stream);

/* ================= L2: multi-crop sampler =====================================================
 * Replaces the per-crop Python loop of slice_imgs (aphantasia/utils.py:243-253) + transforms_fast
 * (aphantasia/transforms.py:165-170): bicubic(A=-0.75, align_corners, crop-clamped) -> perspective
 * (bilinear, zeros, x coverage) -> erase -> rotate (bilinear, zeros, x coverage) -> normalise.
 * canvas [3,H,W]; the sampling frame is the canvas wrap-padded by (pad_top, pad_left)
 * ('over*' aligns, utils.py:152-187; 0,0 otherwise); table: DEVICE [S, APH_CROP_PARAM_FLOATS];
 * out [S,3,size,size] ([S,3,size+8,size+8] for APH_TF_CUSTOM / APH_TF_ELASTIC). size <= 224, the largest crop side
 * the image encoders take; the frame may have any size.                                                             */
int aph_sample_fwd(const float* canvas, int H, int W, int pad_top, int pad_left,
                   const float* table, int S, int size, int kind, float* out, void* stream);
/* Same, and the last stage also writes the batch as the encoder's patch operand (bf16, patch-major: see
 * aph_vit_patch_operand below); the output side (size, or size + 8) must be a multiple of patch, or lie in
 * [res, res + patch) of an encoder with input resolution res = grid * patch: then the operand is the top-left res x res
 * window, as conv1 reads it. The operand is written for every frame size and transform kind:
 * *patches_written = 1 on success.                                                                                   */
int aph_sample_fwd_patches(const float* canvas, int H, int W, int pad_top, int pad_left,
                           const float* table, int S, int size, int kind, float* out,
                           void* patches_bf16, int patch, int* patches_written, void* stream);
/* grad_out [S,3,size,size] -> grad_canvas [3,H,W] (zeroed here, then accumulated), every contribution multiplied by
 * gscale: 1 on one GPU, the weight S_local / S of this rank's shard in the all-reduced gradient under torchrun (folded
 * into the scatter instead of a separate pass over the canvas).                                     */
int aph_sample_bwd_scaled(const float* grad_out, int H, int W, int pad_top, int pad_left,
                          const float* table, int S, int size, int kind, float gscale, float* grad_canvas, void* stream);

/* HOST function (no GPU work): exact native replay of the reference's per-crop random draws (utils.py:244-247,
 * torchvision RandomPerspective/RandomErasing.get_params, transforms.py:75) continuing torch's CPU generator
 * (torch_state = the torch.get_rng_state() blob, updated in place) and NumPy's legacy MT19937 (np_key[624], *np_pos,
 * updated in place). rnd_size/offx/offy are the [count] vectors slice_imgs draws first (utils.py:222-228).
 * Writes tables [n_imgs][count][APH_CROP_PARAM_FLOATS] (HOST memory).                                              */
int aph_rng_crop_tables(uint8_t* torch_state, int64_t torch_state_bytes, uint32_t* np_key, int32_t* np_pos,
                        const float* rnd_size, const float* rnd_offx, const float* rnd_offy, int count,
                        int H, int W, int frame_h, int frame_w, int size, int kind, float macro, int n_imgs,
                        float* tables);

/* ================= L1: CLIP ViT image encoder (B/32, B/16, L/14) ==================================
 * Replaces clip.model.CLIP.encode_image / VisionTransformer.forward (third-party OpenAI clip; call
 * sites clip_fft.py:216,254,276) and its autograd data-gradient. Weights are frozen: no weight
 * gradients are computed (the reference computes and discards them, clip_fft.py:293-295).           */
typedef struct aph_vit aph_vit;
typedef struct {
  int32_t patch;      /* 32, 16 or 14 (any even patch)              */
  int32_t width;      /* 768 (1024 for ViT-L/14; also 128, 256)     */
  int32_t layers;     /* 12 (24)                                    */
  int32_t heads;      /* 12 (16) (head dim must be 64)              */
  int32_t out_dim;    /* 512 (768)                                  */
  int32_t res;        /* input resolution, 224                      */
  int32_t max_batch;  /* largest S a call will pass                 */
  int32_t reserved;
} aph_vit_config;
int aph_vit_create(aph_vit** vit, const aph_vit_config* cfg);
int aph_vit_destroy(aph_vit* vit);
/* One tensor of the OpenAI state dict, by its key ("visual.conv1.weight", "visual.transformer.
 * resblocks.3.attn.in_proj_weight", ...), fp32 DEVICE pointer; converted/transposed to the packed
 * bf16 operand layout on device. aph_vit_finalize checks every tensor arrived.                     */
int aph_vit_load_tensor(aph_vit* vit, const char* key, const float* data, int64_t numel, void* stream);
int aph_vit_finalize(aph_vit* vit);
/* images [S,3,res,res] fp32 (already normalised) -> emb [S,out_dim] fp32. save_for_bwd 0/1.        */
int aph_vit_fwd(aph_vit* vit, const float* images, int S, float* emb, int save_for_bwd, void* stream);
/* Patch operand hand-over (SURVEY 2.4 k10-k12: the sampler emits the patch-major bf16 A operand of conv1, replacing the
 * fp32 round trip x.type(dtype) -> conv1's im2col of the reference's clip/model.py VisionTransformer.forward):
 * aph_vit_patch_operand returns the handle's operand buffer [S*grid*grid, patch_k(patch)] bf16 (row = s*grid*grid + gy*grid + gx,
 * col = c*patch*patch + py*patch + px) for aph_sample_fwd_patches to fill; aph_vit_fwd_prepatched then runs the forward on it.
 * The row stride patch_k(p) is 3*p*p rounded up to a multiple of 128 (3072 for p = 32, 768 for p = 16, 640 for p = 14); the
 * columns from 3*p*p on are zero, set once at create and written by no one.                                                   */
int aph_vit_patch_operand(aph_vit* vit, int S, void** patches_bf16, int* patch, int* grid);
int aph_vit_fwd_prepatched(aph_vit* vit, int S, float* emb, int save_for_bwd, void* stream);
/* grad_emb [S,out_dim] -> grad_images [S,3,res,res] (overwritten). Uses activations of the last
 * aph_vit_fwd(save_for_bwd=1) with the same S.                                                     */
int aph_vit_bwd(aph_vit* vit, const float* grad_emb, int S, float* grad_images, void* stream);
/* The same for images of side `side` in [res, res + patch): conv1 (kernel = stride = patch, no padding) reads only the
 * top-left res x res window, so the forward reads that window through a row stride and the backward writes grad_images
 * [S,3,side,side] with an exactly zero margin (rows and columns >= res). side == res is aph_vit_fwd / aph_vit_bwd.     */
int aph_vit_fwd_sized(aph_vit* vit, const float* images, int S, int side, float* emb, int save_for_bwd, void* stream);
int aph_vit_bwd_sized(aph_vit* vit, const float* grad_emb, int S, int side, float* grad_images, void* stream);
/* bytes of device memory owned by the handle (weights + activation arena)                          */
int64_t aph_vit_bytes(const aph_vit* vit);

/* ================= L1: CLIP ResNet image encoder (RN50, RN101) ===================================
 * Replaces clip.model.ModifiedResNet.forward (third-party OpenAI clip) in eval mode and its data gradient: stem (three 3x3
 * convolutions, the first of stride 2, each + BatchNorm + ReLU; avgpool 2), four stages of bottlenecks (layers[i] blocks of
 * planes 64 << i, expansion 4, stride 2 in the first block of stages 2-4 as an average pool), the attention pool (mean token +
 * 49 map tokens + positional embedding, 32-head attention queried by token 0, c_proj). No weight gradients.
 * Keys of aph_rn_load_tensor are the OpenAI ones without "visual." after folding every BatchNorm (eps 1e-5, running statistics)
 * into its convolution (aphantasia_b200.clip.fold_resnet_state_dict): "conv{1,2,3}.weight" / ".bias" (conv1 [32,3,3,3]; conv2,
 * conv3 zero-padded to [64,64,3,3], conv2's bias to [64]), "layer{i}.{j}.conv{1,2,3}.weight" / ".bias",
 * "layer{i}.{j}.downsample.weight" / ".bias" (the 1x1 convolution of downsample.1 folded with downsample.2),
 * "attnpool.positional_embedding", "attnpool.qkv.weight" [3*2048, 2048] = [q_proj; k_proj; v_proj] and "attnpool.qkv.bias",
 * "attnpool.c_proj.weight" / ".bias". aph_rn_finalize checks every tensor arrived.
 * Device bytes (aph_rn_bytes) = weights + arena, S = max_batch, D = 2048, O = out_dim, sizes of a side-254 input
 * (h1 = 127 after the stem's convolutions, h0 = 63 after its pool; block b has input map hin_b, output map hout_b = hin_b /
 * stride_b, cin_b input channels, P_b planes, E_b = 4 P_b):
 *   weights  4 (864 + 32 + 2*64) + 2 * 2 * 2 * 9 * 64 * 64
 *            + sum_b [2 * 2 (P cin + E P (+ E cin if downsample)) + 2 * 2 * 9 P^2 + 4 (2 P + E (+ E if downsample))]
 *            + 4 * 50 D + 2 * 2 * 3 D^2 + 4 * 3 D + 2 * 2 O D + 4 O
 *   arena    2 [S (3 h1^2 64 + h0^2 64) + sum_b S (2 hin_b^2 P_b + hout_b^2 E_b) + 6 S emax + 10 * 50 S D + S O] + 4 S O
 *            emax = max(h1^2 64, max_b hin_b^2 max(cin_b, P_b), max_b hout_b^2 E_b)                                      */
typedef struct aph_rn aph_rn;
typedef struct {
  int32_t layers[4];  /* (3, 4, 6, 3) RN50, (3, 4, 23, 3) RN101         */
  int32_t width;      /* 64                                            */
  int32_t heads;      /* 32 (head dim 64)                              */
  int32_t out_dim;    /* 1024 (RN50), 512 (RN101)                      */
  int32_t res;        /* input resolution, 224                         */
  int32_t max_batch;  /* largest S a call will pass                    */
  int32_t reserved;
} aph_rn_config;
int aph_rn_create(aph_rn** rn, const aph_rn_config* cfg);
int aph_rn_destroy(aph_rn* rn);
int aph_rn_load_tensor(aph_rn* rn, const char* key, const float* data, int64_t numel, void* stream);
int aph_rn_finalize(aph_rn* rn);
/* x [S,3,side,side] fp32 (normalised crops), 223 <= side <= 254 (the sides whose final map is 7 x 7; the whole crop is read)
 * -> emb [S,out_dim]. save_for_bwd 0/1.                                                                                   */
int aph_rn_fwd(aph_rn* rn, const float* x, int S, int side, float* emb, int save_for_bwd, void* stream);
/* grad_emb [S,out_dim] -> grad_x [S,3,side,side] (overwritten), from the last aph_rn_fwd(save_for_bwd = 1) of the same S, side. */
int aph_rn_bwd(aph_rn* rn, const float* grad_emb, int S, int side, float* grad_x, void* stream);
int64_t aph_rn_bytes(const aph_rn* rn);
/* Test entries of the tower's own kernels on caller buffers (bf16 NHWC activations):
 * aph_rn_stem_test: stem conv 1, weight fp32 [32,3,3,3], bias [32], h = (side - 1) / 2 + 1. fwd = 1: in = crops fp32
 *   [N,3,side,side] -> out bf16 [N,h,h,64] = relu(conv + bias) in channels 0-31, zero above; fwd = 0: in = dz bf16 [N,h,h,64]
 *   (channels 0-31 read) -> out fp32 [N,3,side,side].
 * aph_rn_pool_test: 2x2 average pool (floor), C % 8 == 0. fwd = 1: out = pool(x) [N,H/2,W/2,C]; fwd = 0: x = dy [N,H/2,W/2,C]
 *   -> out [N,H,W,C] = its adjoint, selected by mask [N,H,W,C] > 0 unless mask is NULL.
 * aph_rn_tokens_test: fwd = 1: in = x bf16 [S*49,C], aux = pos fp32 [50,C] -> out bf16 [S*50,C] (row 0 the mean of the 49 rows,
 *   + pos); fwd = 0: in = dtok bf16 [S*50,C], aux = x -> out [S*49,C] = x > 0 ? dtok[1 + i] + dtok[0] / 49 : 0.
 * aph_rn_saved_test: the last saved forward's ReLU outputs (handle memory, valid until the next forward), bf16 NHWC: k = 0..2
 *   the stem's [S,h,h,64], then for block b (stages in order) 3 b + 3 / 3 b + 4 its conv1 / conv2 outputs [S,hin,hin,P] and
 *   3 b + 5 its output [S,hout,hout,4 P]; *numel their element count.
 * aph_gemm_rn_epi_test: the encoder GEMM with the ResNet epilogues (N = 64 or a multiple of 128): relu = 1: out_bf16 =
 *   relu(acc + bias [+ resid_bf16]); relu = 0: out_bf16 = mask > 0 ? acc [+ resid_bf16] : 0 (bias unused). NULL = absent.  */
int aph_rn_saved_test(aph_rn* rn, int k, void** ptr, int64_t* numel);
int aph_rn_stem_test(int fwd, const void* in, const float* weight, const float* bias, void* out, int N, int side, void* stream);
int aph_rn_pool_test(int fwd, const void* x, const void* mask, void* out, int N, int H, int W, int C, void* stream);
int aph_rn_tokens_test(int fwd, const void* in, const void* aux, void* out, int S, int C, void* stream);
int aph_gemm_rn_epi_test(const void* A, const void* B, int M, int N, int K, const float* bias, const void* resid_bf16,
                         const void* mask, int relu, void* out_bf16, void* stream);

/* ================= CLIP text encoder (forward only) ===========================================
 * Replaces clip.model.CLIP.encode_text (third-party OpenAI clip; call site clip_fft.py:150), run once per prompt
 * before the optimisation loop: token_embedding[ids] + positional_embedding -> layers x pre-LN residual block with
 * CAUSAL attention -> ln_final(x[s, argmax(ids[s])]) @ text_projection. Same kernels as the image tower.          */
typedef struct aph_text aph_text;
typedef struct {
  int32_t width;      /* 512 (multiple of 128, <= 1024)              */
  int32_t layers;     /* 12                                           */
  int32_t heads;      /* 8 (head dim must be 64)                      */
  int32_t out_dim;    /* 512 (multiple of 128)                        */
  int32_t context;    /* 77 (<= 112)                                  */
  int32_t vocab;      /* 49408                                        */
  int32_t max_batch;  /* largest n a call will pass                   */
  int32_t reserved;
} aph_text_config;
int aph_text_create(aph_text** t, const aph_text_config* cfg);
int aph_text_destroy(aph_text* t);
/* One tensor of the OpenAI state dict by its key (token_embedding.weight, positional_embedding,
 * transformer.resblocks.N.{ln_1,attn,ln_2,mlp}.*, ln_final.weight / bias, text_projection), fp32 DEVICE pointer.
 * token_embedding stays fp32 on the device; the layer matrices are packed to bf16. aph_text_finalize checks
 * every tensor arrived.                                                                                          */
int aph_text_load_tensor(aph_text* t, const char* key, const float* data, int64_t numel, void* stream);
int aph_text_finalize(aph_text* t);
/* tokens int64 [n, context] DEVICE -> emb [n, out_dim] fp32. Pooling row = first position of the largest id
 * (torch.argmax). Ids outside [0, vocab) read no memory out of bounds (they embed as zeros); callers reject them. */
int aph_text_fwd(aph_text* t, const int64_t* tokens, int n, float* emb, void* stream);
/* bytes of device memory owned by the handle (weights + activations)                              */
int64_t aph_text_bytes(const aph_text* t);

/* Stand-alone wgmma GEMM used by the encoder (exported for tests / profiling):
 * C[M,N] (fp32) = A[M,K] (bf16, row-major) . B[N,K]^T (bf16, row-major). K % 64 == 0, N % 128 == 0. */
int aph_gemm_bf16_tn(const void* A, const void* B, float* C, int M, int N, int K, void* stream);

/* Test entries. aph_gemm_epi_test: the same GEMM with the encoder's fused epilogues on caller-supplied operands
 * (NULL = unused; the combination selects the kind as the encoder's own calls do: +bias, QuickGELU saving the
 * pre-activation (act=1, out_pre), x gelu'(gelu_in), +fp32 resid, fp32 / bf16 outputs, NCHW un-patchify).
 * bf16 operands of the epilogue (out_bf16, out_pre, gelu_in) must be 16-byte aligned.
 * aph_gemm_variant_launches: launches so far of kernel variant 0 (the small-problem kernel) or 1 (the large-problem kernels:
 * ping-pong 128x128 tiles for short K, cooperative 128x256 tiles for long K) with epilogue kind epi
 * (0 f32, 1 bf16, 2 bias-bf16, 3 bias-gelu, 4 bias-resid, 5 gelu-grad, 6 un-patchify; -1 = any).                                                             */
int aph_gemm_epi_test(const void* A, const void* B, int M, int N, int K, const float* bias, const float* resid,
                      const void* gelu_in, int act, float* out_f32, void* out_bf16, void* out_pre,
                      int unpatch_p, int unpatch_g, void* stream);
/* aph_gemm_epi_strided_test: the same without un-patchify, with row strides in elements (0 = dense) for A (lda), the residual
 * (ld_resid) and the outputs and gelu_in (ld_out), as the encoder's last block reads and writes its class-token rows.
 * Strides must be multiples of 16 bytes; rows between the strided output rows are not written.                      */
int aph_gemm_epi_strided_test(const void* A, int lda, const void* B, int M, int N, int K, const float* bias,
                              const float* resid, int ld_resid, const void* gelu_in, int act, float* out_f32,
                              void* out_bf16, void* out_pre, int ld_out, void* stream);
int64_t aph_gemm_variant_launches(int variant, int epi);
/* aph_attn_test: the encoder's attention core on caller operands. qkv bf16 [S*T, 3*D] (q | k | v), D = 64*heads.
 * fwd = 1: out bf16 [S*T, D]; fwd = 0: dout bf16 [S*T, D] in, out = dqkv bf16 [S*T, 3*D]. causal = 0 runs the image
 * tower's dispatch (T <= 256), causal = 1 the text tower's causal forward (T <= 112; there is no causal backward).
 * Unsupported shapes return an error and launch nothing.
 * aph_attn_long_test: the streaming attention kernels the image tower runs for T > 256 (ViT-L/14: T = 257), on the same
 * operands as aph_attn_test with causal = 0, for any T >= 1.
 * aph_ln_fwd_test: k_ln_fwd on x fp32 [rows, D] (row stride D) -> y bf16 [rows, D], mean / rstd fp32 [rows].
 * aph_ln_bwd_test: k_ln_bwd with dy fp32 (dy_bf16 = 0) or bf16 (dy_bf16 = 1) [rows, D]; mode 0: dx (+)= LN'(dy) (fp32 dx and
 * bf16 dx_bf16, accumulate = 1 adds to dx); mode 1: dx = LN'(dy) + dcls[s] on rows s*T (dcls fp32 [rows/T, D]); mode 2:
 * the non-class rows into dx_bf16 = dtok bf16 [rows/T*(T-1), D], dx unused. D in {128, 256, 512, 768, 1024}.            */
int aph_attn_test(int fwd, int causal, const void* qkv, const void* dout, void* out, int S, int T, int D, int heads, void* stream);
int aph_attn_long_test(int fwd, const void* qkv, const void* dout, void* out, int S, int T, int D, int heads, void* stream);
int aph_ln_fwd_test(const float* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd, int rows, int D,
                    void* stream);
int aph_ln_bwd_test(const void* dy, int dy_bf16, const float* x, const float* mean, const float* rstd, const float* gamma, float* dx,
                    void* dx_bf16, int rows, int T, int D, int mode, int accumulate, const float* dcls, void* stream);

/* Profiling aid: enable=1 records a CUDA-event pair around every GEMM launch of this library; enable=0 stops and returns
 * the summed kernel time (ms), FLOPs (sum of 2MNK) and launch count since enabling (bench.py's roofline).            */
int aph_prof_gemm(int enable, double* total_ms, double* total_flops, int* launches);

/* ================= L1: similarity loss ========================================================
 * Replaces sim_func(v1, v2, type) for type in {None/'cossim', 'mix'} (aphantasia/utils.py:276-282,
 * 295). v1 [n1,D] with n1 in {1,S}; v2 [S,D]. value (device scalar) = mean_s f(v1, v2_s).
 * grad_v1 / grad_v2 may be NULL; they receive d value / d v (not yet multiplied by the upstream
 * gradient).                                                                                       */
int aph_sim_fwd(const float* v1, int n1, const float* v2, int S, int D, int kind,
                float* value, float* grad_v1, float* grad_v2, void* stream);

/* ---- optional loss heads (SURVEY.md 8 row f4) ---------------------------------------------------
 * derivat(img, mode='naiv') (aphantasia/utils.py:256-268; clip_fft.py:271-272 --sharp): img [C,H,W];
 * value = 0.5*(mean|d/dx| + mean|d/dy|); sums = double[2] device scratch. The backward multiplies by the
 * upstream gradient read from a DEVICE scalar.                                                      */
int aph_derivat_fwd(const float* img, int C, int H, int W, double* sums, float* value, void* stream);
int aph_derivat_bwd(const float* img, int C, int H, int W, const float* upstream, float* grad_img, void* stream);
/* derivat(img, mode='sobel') (aphantasia/utils.py:262-264; cppn.py:291-292 --sharp): mean |kornia spatial_gradient(img)|, the
 * Sobel pair normalised by 1/8 with replicate padding, over the 2*C*H*W outputs. img [C,H,W] (C = N*channels); sums = double[1]
 * device scratch. The backward multiplies by the upstream gradient read from a DEVICE scalar; sign(0) = 0.            */
int aph_derivat_sobel_fwd(const float* img, int C, int H, int W, double* sums, float* value, void* stream);
int aph_derivat_sobel_bwd(const float* img, int C, int H, int W, const float* upstream, float* grad_img, void* stream);
/* Linear head on the embeddings: the LAION aesthetic predictor of --aest is nn.Linear(D, 1)
 * (aphantasia/utils.py:402-413; clip_fft.py:255-256). out[s] = <emb_s, w> + b[0] (b may be NULL).   */
int aph_head_fwd(const float* emb, int S, int D, const float* w, const float* b, float* out, void* stream);
int aph_head_bwd(const float* grad_out, const float* w, int S, int D, float* grad_emb, void* stream);

/* ---- LPIPS image-composition loss (clip_fft.py --sync: lpips.LPIPS(net='vgg'), clip_fft.py:220,270) --------------------
 * lpips v0.1, net='vgg', lpips=True, spatial=False: scaling layer, VGG16 features[0:30] (13 conv3x3 + ReLU, 4 max-pools), per-tap
 * unit-normalised features, squared difference weighted by the tap's lin weights, spatial mean, sum over the 5 taps.
 * Keys of aph_lpips_load_tensor (fp32 DEVICE data): torchvision's "features.{i}.weight" [Co,Ci,3,3] / "features.{i}.bias" for
 * i in {0,2,5,7,10,12,14,17,19,21,24,26,28}, and lpips' "lin{t}.model.1.weight" [1,C,1,1], t = 0..4. The 3x3 weights are packed
 * once, to bf16 [Co, 9 Ci] for the forward and [Ci, 9 Co] (flipped) for the data gradient.                                   */
typedef struct aph_lpips aph_lpips;
int aph_lpips_create(aph_lpips** h);
int aph_lpips_destroy(aph_lpips* h);
int aph_lpips_load_tensor(aph_lpips* h, const char* key, const float* data, int64_t numel, void* stream);
int aph_lpips_finalize(aph_lpips* h);
/* in0, in1 [N,3,H,W] (H, W >= 16) -> out [N] = LPIPS(in0[n], in1[n]); normalize = 1 maps inputs from [0,1] to [-1,1].
 * The features of in1 are cached under ref_key (non-zero; 0 = do not reuse): in1 may be NULL when ref_key matches the cached
 * features of the same N, H, W, and then no reference pass runs. save_for_bwd = 1 keeps the activations of in0;
 * *generation (may be NULL) receives this forward's stamp. Every forward voids the activations saved by earlier ones.      */
int aph_lpips_fwd(aph_lpips* h, const float* in0, const float* in1, uint64_t ref_key, int N, int H, int W, int normalize,
                  float* out, int save_for_bwd, int64_t* generation, void* stream);
/* grad_out [N] DEVICE -> grad_in0 [N,3,H,W] (overwritten). Fails, launching nothing, if `generation` is not the last forward's
 * or that forward did not save.                                                                                            */
int aph_lpips_bwd(aph_lpips* h, const float* grad_out, int64_t generation, float* grad_in0, void* stream);
/* Test entries on caller buffers (bf16 NHWC activations):
 * aph_lpips_conv_test: one 3x3 layer, weight fp32 [Cout,Cin,3,3] packed as the loader does. fwd = 1: x [N,H,W,Cin] ->
 *   out = relu(conv(x) + bias) [N,H,W,Cout]; fwd = 0: x = dy [N,H,W,Cout] -> out = dx [N,H,W,Cin], with mask (NULL = none)
 *   [N,H,W,Cin]: out = mask > 0 ? dx : 0. Cin, Cout multiples of 64.
 * aph_lpips_conv0_test: conv1_1 (3 -> 64, fp32). fwd = 1: in = image fp32 [N,3,H,W] -> out bf16 [N,H,W,64] (ReLU output,
 *   after the scaling layer); fwd = 0: in = dz bf16 [N,H,W,64] -> out fp32 [N,3,H,W].
 * aph_lpips_pool_test: 2x2 max-pool, C % 8 == 0. fwd = 1: out = pool(x); fwd = 0: out [N,H,W,C] = adjoint of dy [N,H/2,W/2,C]. */
int aph_lpips_conv_test(int fwd, const void* x, const float* weight, const float* bias, const void* mask, void* out, int N, int H,
                        int W, int Cin, int Cout, void* stream);
int aph_lpips_conv0_test(int fwd, const void* in, const float* weight, const float* bias, void* out, int N, int H, int W,
                         int normalize, void* stream);
int aph_lpips_pool_test(int fwd, const void* x, const void* dy, void* out, int N, int H, int W, int C, void* stream);

/* ================= step glue ==================================================================
 * torch.optim.Adam(betas=(b1,b2)) / AdamW(..., weight_decay, amsgrad) single-tensor update of step `step` >= 1
 * (clip_fft.py:108-115,295), bias-corrected: weight_decay != 0 decays p by 1 - lr * weight_decay first (AdamW);
 * vmax != NULL is AMSGrad's running maximum of v, and the denominator uses it. The trailing arguments come after the
 * stream so that callers of the plain form bind unchanged (the Python binding passes 0 / NULL for them).           */
int aph_adam_step(float* p, const float* g, float* m, float* v, int64_t n,
                  float lr, float b1, float b2, float eps, int step, void* stream,
                  float weight_decay, float* vmax);

/* SURVEY.md 8 row f2: aph_synth_fft_bwd with the Adam update of the spectrum fused into its last pass (the data
 * gradient dP is in registers there): params / m / v (/ vmax) [3,H,Wh,2] are updated in place; grad_params may be NULL
 * (nothing is written) or receives dP as aph_synth_fft_bwd does. Same arithmetic as aph_adam_step.              */
int aph_synth_fft_bwd_adam(aph_fft_plan* plan, const float* grad_out, const float* out, const float* x_raw,
                           double* stats, const float* scale, float contrast, const float* colmat_host,
                           int apply_sigmoid, float* grad_params, float* params, float* m, float* v,
                           float lr, float b1, float b2, float eps, int step, void* stream,
                           float weight_decay, float* vmax);

/* ================= multi-GPU exchange (SURVEY.md 8e) ==========================================
 * In-place all-reduce(SUM) of a fp32 buffer in SYMMETRIC memory (the canvas gradient dRGB [3,H,W], replacing the
 * single NCCL all-reduce of the path): one kernel, two shots over NVSwitch multicast (multimem.ld_reduce / multimem.st;
 * mc_ptr = multicast address) or, with mc_ptr == 0, over the peers' mapped pointers. peer_ptrs: HOST array[world] of
 * every rank's device mapping of the buffer; signal_pads_dev: DEVICE array[world] of pointers to zero-initialised
 * uint32 signal pads (>= 32*world words each); numel % 4 == 0. err_flag (device int) is set if a barrier timed out.  */
int aph_allreduce_sym(uint64_t mc_ptr, const uint64_t* peer_ptrs, const uint64_t* signal_pads_dev, int rank, int world,
                      int64_t numel, int* err_flag, void* stream);

/* number of kernels this library has launched since load (bench.py's gpu_launches)                 */
int64_t aph_launch_count(void);

/* device bytes this library holds right now: handles, plans, their scratch, and stream-ordered temporaries not yet freed.
 * Unlike cudaMemGetInfo it counts no other process's memory, so a test can check that a destroy returns everything.   */
int64_t aph_device_bytes(void);

#ifdef __cplusplus
}
#endif
#endif /* APHB200_H_ */

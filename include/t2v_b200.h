/* t2v_b200 -- C ABI of the GPU-native (sm_90a) text2video denoising path.
 *
 * The reference (kabachuha/sd-webui-text2video) has NO FFI boundary: its hot path is plain Python that calls
 * PyTorch library kernels.  This header is the boundary a maintainer would bind instead (ctypes stubs in
 * INTEGRATION.md); every entry point names the reference call it replaces (paths relative to
 * /root/reference/scripts).
 *
 * Conventions (mirroring the Python contract, SURVEY.md section 8b):
 *   - plain pointers and sizes only; device pointers unless stated otherwise; the CALLER owns every tensor passed
 *     in, the library owns only its packed-weight and workspace arenas (freed by *_destroy)
 *   - all work is enqueued asynchronously on `stream` (a cudaStream_t passed as void*), no hidden synchronisation
 *   - return value 0 = success, negative = error (t2v_last_error() gives the text); the Python layer raises
 *     RuntimeError so failures surface as exceptions exactly like the reference (t2v_helpers/render.py:35-37)
 *   - a handle is bound to one device and is not thread-safe (the webui serialises callers, text2vid.py:82)
 */
#ifndef T2V_B200_H
#define T2V_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------ library */
int t2v_init(int device);                 /* selects the device, resolves driver entry points, sizes grids */
const char* t2v_last_error(void);
int t2v_num_sms(void);
const char* t2v_version(void);

/* ------------------------------------------------------------------------------------------ denoiser
 * replaces modelscope/t2v_model.py::UNetSD (ctor :98-326, forward :386-501).                            */
typedef struct t2v_unet t2v_unet;

typedef struct {
    int in_dim, dim, context_dim, out_dim;
    int dim_mult[8];
    int n_mult;
    int num_heads;        /* heads of the stem TemporalTransformer (:171-179) */
    int head_dim;         /* must be 64 */
    int num_res_blocks;
    float attn_scales[8];
    int n_attn_scales;
    int arch;              /* 0: ModelScope UNetSD (modelscope/t2v_model.py:98-501)
                            * 1: VideoCrafter UNetModel (videocrafter/lvdm/models/modules/openaimodel3d.py:281-670; dim =
                            *    model_channels, dim_mult = channel_mult, attn_scales = 1/attention_resolutions, head width =
                            *    channels / num_heads (head_dim ignored), state_dict keys of `model.diffusion_model.*`) */
    int temporal_length;   /* arch 1: RelativePosition(max_relative_position = temporal_length), tables [2*L+1, d] */
} t2v_unet_config;

int t2v_unet_create(const t2v_unet_config* cfg, t2v_unet** out);
void t2v_unet_destroy(t2v_unet* u);
/* Hands one parameter of the reference state_dict (key names of SURVEY.md appendix D, e.g.
 * "input_blocks.1.0.in_layers.2.weight") to the library, which packs it into its own layout.
 * `data` is a DEVICE pointer to a contiguous tensor of `dtype` (0 = fp16, 1 = fp32) with `ndim` dims.
 * Replaces load_state_dict(strict=True) at modelscope/t2v_pipeline.py:95-101 (and is what the LoRA merger's
 * re-assigned .weight tensors are re-sent through, stable_lora/scripts/lora_processor.py:236-242).        */
int t2v_unet_set_param(t2v_unet* u, const char* name, const void* data, int dtype, int ndim, const int64_t* shape,
                       void* stream);
/* Number of parameters still missing (0 => ready); fills `name_out` with one missing key if non-null. */
int t2v_unet_missing_params(t2v_unet* u, char* name_out, size_t name_cap);
/* Enumerates the expected state_dict: index in [0, count) -> key name + shape (shape has room for 8 dims).
 * Returns the number of expected parameters, or -1 if `index` is out of range.  The Python mirror builds its
 * nn.Module tree (same names, nn.Linear / nn.Conv2d / nn.Conv3d leaves) from this list.                     */
int t2v_unet_param_info(t2v_unet* u, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out);
/* eps = UNetSD.forward(x, t, y) (t2v_model.py:386-459).
 *   x   [B, in_dim, F, h, w]  fp32 (x_is_f32 = 1) or fp16, NCFHW exactly as the samplers hold the latent
 *   t   [B] float32 (host converts int64 timesteps; UniPC already passes floats, uni_pc.py:248)
 *   ctx [B, L, context_dim] fp16
 *   out [B, out_dim, F, h, w] fp16 (out_is_f32 = 0) or fp32                                               */
int t2v_unet_forward(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx, void* out,
                     int out_is_f32, int B, int F, int h, int w, int L, void* stream);
/* t2v_unet_forward with a context batch ctx_B that divides B: ctx [ctx_B, L, context_dim], sample j reads prompt
 * j / (B / ctx_B) -- for n clips guided as one batch, x = [x_1..x_n, x_1..x_n] and ctx = [c, uc] (ctx_B = 2).  The
 * cross-attention K/V GEMMs project only the ctx_B * L distinct prompt rows, once per forward.  ctx_B = B is exactly
 * t2v_unet_forward (same plan); ctx_B < B has a plan of its own.  Not available on a frame-sharded denoiser.          */
int t2v_unet_forward_ctx(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx, int ctx_B, void* out,
                         int out_is_f32, int B, int F, int h, int w, int L, void* stream);
/* eps = UNetModel.forward(x, t, context, features_adapter) (videocrafter/lvdm/models/modules/openaimodel3d.py:632-670), arch 1
 * only: feature i is added to h after input block id with (id + 1) % 3 == 0 (the i-th such block, counting from 0), before h is
 * pushed on the skip stack.  feats[i] is a device pointer to [feats_B, F, h_i, w_i, C_i] fp16, channels-last: the
 * reference's `b c t h w` feature permuted to (b, t, h, w, c), with h_i, w_i, C_i those of h at that block.  Sample j of the
 * forward reads feature sample j % feats_B (feats_B = 1: broadcast; B = 2 feats_B: a batched cond / uncond pair).
 * n_feats must equal the number of such blocks and B a multiple of feats_B.  The features are staged per forward (copied
 * device to device); the plan of a shape with features is separate from the plan without, which t2v_unet_forward keeps
 * using unchanged.  Other arguments as t2v_unet_forward.                                                          */
int t2v_unet_forward_adapter(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx,
                             const void* const* feats, int n_feats, int feats_B, void* out, int out_is_f32, int B, int F, int h,
                             int w, int L, void* stream);
/* 2*MAC flop count of one forward at this shape (for roofline reporting). */
double t2v_unet_flops(t2v_unet* u, int B, int F, int h, int w, int L);
/* Activation-slab bytes the plan of this shape allocates (host only: the same dry pass as t2v_unet_flops). */
int t2v_unet_plan_bytes(t2v_unet* u, int B, int F, int h, int w, int L, size_t* arena);
/* Both of the above for the plan of a forward with context batch ctx_B (t2v_unet_forward_ctx), host only; *cached = 1 if the
 * denoiser holds that plan for its current weights already (a forward then allocates nothing).  flops, cached may be null. */
int t2v_unet_plan_info(t2v_unet* u, int B, int ctx_B, int F, int h, int w, int L, size_t* arena, double* flops, int* cached);
int t2v_unet_num_launches(t2v_unet* u);
/* Measurement aid: replays the plan of this shape once (inputs = whatever the last forward left in the staging
 * buffers) with a CUDA-event pair around every launch on `stream` and sums per kernel family:
 *   out[3k + 0] = milliseconds, out[3k + 1] = algorithmic flop, out[3k + 2] = launches, k = 0 implicit-GEMM (wgmma),
 *   1 attention, 2 group/layer norm, 3 glue; out[12] = total ms.  Synchronises the stream (bench/tests only).   */
int t2v_unet_profile(t2v_unet* u, int B, int F, int h, int w, int L, void* stream, double* out13);
/* copies an internal activation (debug / parity taps): name = reference module path (e.g. "input_blocks.1.0"),
 * dst receives [(B F), C, h, w] fp16 as the reference module returns it. Returns element count or <0. */
long long t2v_unet_read_tap(t2v_unet* u, const char* name, void* dst, long long cap_elems, void* stream);
int t2v_unet_enable_taps(t2v_unet* u, int on);
/* shape of a tap of the most recent plan: rows x C token matrix viewed as [(rows / (h w)), C, h, w].  A frame-sharded clip
 * records spatial modules frame-sharded (this rank's frames, full h x w) and temporal modules pixel-sharded (all frames,
 * h = 1, w = this rank's pixel count).  Returns 0, or -1 if the tap does not exist. */
int t2v_unet_tap_info(t2v_unet* u, const char* name, long long* rows, int* C, int* h, int* w);

/* ------------------------------------------------------------------------------------------ LoRA hot-merge
 * replaces StableLoraProcessor.process_lora's weight surgery (stable_lora/stable_utils/lora_processor.py:50-96, :202-246):
 * instead of re-assigning `m.weight = nn.Parameter(W +- alpha * B @ A)` and re-shipping / re-packing the whole model, the
 * low-rank update is applied to the library's own copy of ONE weight,
 *     W <- fp16(W + fp16(fp16(B @ A) * alpha))        (the reference's roundings under autocast; several merges accumulate)
 * and only the packed variants derived from it (tap-major conv layout, fused q|k|v, GEGLU interleave, LayerNorm-folded
 * copies) are rebuilt in place -- buffer addresses, plans and captured CUDA graphs stay valid, the next forward just uses the
 * new weights.  lora_A [rank, cols] and lora_B [out, rank] are fp16 device pointers, cols = in * kernel taps of the weight;
 * temporal_mean = 1 for Conv3d (3,1,1) weights: lora_A has in * 9 columns, the product is viewed [out, in, 3, 3, 1] and
 * averaged over the second kernel axis (:86-94).  t2v_unet_lora_clear restores every merged weight from its base copy:
 * bit-identical to never having merged (the reference's `-=` undo leaves fp16 rounding residue; this does not).        */
int t2v_unet_lora_merge(t2v_unet* u, const char* weight_name, const void* lora_A, const void* lora_B, int rank, float alpha,
                        int temporal_mean, void* stream);
int t2v_unet_lora_clear(t2v_unet* u, void* stream);
int t2v_unet_lora_merged(t2v_unet* u);          /* number of weights currently carrying a merge */

/* ------------------------------------------------------------------------------------------ VideoCrafter LoRA
 * replaces net_load_lora / change_lora / net_load_lora_v2 / change_lora_v2 (videocrafter/lvdm/models/modules/lora.py:620-755):
 * `weight.data += alpha * torch.mm(up, down)` on ONE weight of a handle (UNet, VAE, CLIP text tower, depth adapter), in the
 * library's own copy,
 *     W <- fp16(float(W) + alpha * sum_r float(up[o, r]) * float(down[r, j]))     (fp32 product and sum, ONE rounding)
 * followed by the same in-place re-pack as t2v_unet_lora_merge: plans and captured graphs stay valid.  up [out, rank] and
 * down [rank, cols] are device pointers, both fp16 (dtype 0) or both fp32 (dtype 1; LoRA checkpoints are usually fp32 and
 * are not rounded first); cols = the weight's elements per output row (a 1x1 conv's input channels; the caller squeezes 4-D
 * factors).  The reference's `remove=True` (`-=`) is alpha negated: a subtraction in fp16 storage leaves up to one fp16 ulp
 * of residue per element.  The first merge into a weight keeps a base copy; *_lora_restore copies it back into that one
 * weight and frees it (net_load_lora_v2's origin_weight restore: bit-identical to never merging; a weight without a merge
 * is left as it is), *_lora_clear does so for every weight, *_lora_merged counts the weights carrying a merge.  The UNet's
 * t2v_unet_lora_clear / t2v_unet_lora_merged above serve both merge kinds.                                            */
int t2v_unet_lora_apply(t2v_unet* u, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                        void* stream);
int t2v_unet_lora_restore(t2v_unet* u, const char* weight_name, void* stream);

/* ------------------------------------------------------------------------------------------ frame-sharded clip
 * ONE clip split over the GPUs of a node, one process per GPU (e.g. BASELINE config 4's 125 frames over 8 GPUs).  Frames are
 * independent inside the spatial modules and coupled in TemporalConvBlock_v2 (t2v_model.py:1201-1212), TemporalTransformer
 * (:724, :734-738) and every 5-D GroupNorm; the library keeps activations frame-sharded in the spatial modules, transposes
 * them to a pixel-sharded layout around each temporal module with a kernel that writes straight into the peers' buffers
 * over NVLink (CUDA IPC mappings), and sums the 5-D GroupNorm statistics across ranks inside the statistics kernel.  No
 * NCCL call and no host synchronisation happens inside a forward; the caller's only collective is the exchange of the
 * fixed-size exports below (any byte all-gather: torch.distributed in the Python mirror) once per shape.
 *   1. t2v_unet_shard_setup(u, rank, nranks)                    every rank, once
 *   2. t2v_unet_shard_prepare(u, shape..., &mine)               builds this rank's plan, fills `mine`
 *   3. all-gather the exports in rank order -> all[nranks]
 *   4. t2v_unet_shard_connect(u, shape..., all)                 maps the peers' slabs
 *   5. t2v_unet_forward(u, x_local, ..., F = TOTAL frames ...)  x / out hold this rank's frames [B, C, F_local, h, w];
 *      every rank must issue the same sequence of forwards (the exchange kernels wait for their peers).              */
typedef struct {
    unsigned char comm_handle[64];        /* cudaIpcMemHandle_t of the rank's flag / GroupNorm exchange region */
    unsigned char slab_handle[64];        /* cudaIpcMemHandle_t of the plan's activation slab */
    int rank, nranks;
    int n_exchanges, n_groupnorms;
    long long dst_offset[192];            /* byte offset of every exchange's destination buffer inside the slab */
} t2v_shard_export;
int t2v_unet_shard_setup(t2v_unet* u, int rank, int nranks);
int t2v_unet_shard_prepare(t2v_unet* u, int B, int F, int h, int w, int L, void* stream, t2v_shard_export* out);
int t2v_unet_shard_connect(t2v_unet* u, int B, int F, int h, int w, int L, const t2v_shard_export* all, void* stream);
/* 1 if the plan of this shape exists for the current weights and is connected (a re-shipped parameter or a plan-cache
 * eviction drops the plan: prepare + connect again -- every rank takes the same decision, the inputs are identical) */
int t2v_unet_shard_connected(t2v_unet* u, int B, int F, int h, int w, int L);
/* device-side barrier over the ranks (after connect; all ranks must call it) */
int t2v_unet_shard_barrier(t2v_unet* u, void* stream);
/* this rank's frame range [begin, end) of an F-frame clip and the exchange count of the last forward */
int t2v_unet_shard_info(t2v_unet* u, int F, int* frame_begin, int* frame_end, int* n_exchanges);

/* ------------------------------------------------------------------------------------------ VAE decoder
 * replaces AutoencoderKL.decode (modelscope/t2v_model.py:1646-1649) + ldm Decoder (vendored twin
 * videocrafter/lvdm/models/modules/autoencoder_modules.py:484-596) and the per-frame loop of
 * t2v_pipeline.py:329-355 (all frames batched).                                                           */
typedef struct t2v_vae t2v_vae;
typedef struct {
    int ch;
    int ch_mult[8];
    int n_mult;
    int num_res_blocks;
    int z_channels;
    int out_ch;
    int embed_dim;
} t2v_vae_config;
int t2v_vae_create(const t2v_vae_config* cfg, t2v_vae** out);
void t2v_vae_destroy(t2v_vae* v);
int t2v_vae_set_param(t2v_vae* v, const char* name, const void* data, int dtype, int ndim, const int64_t* shape,
                      void* stream);
int t2v_vae_missing_params(t2v_vae* v, char* name_out, size_t name_cap);
int t2v_vae_param_info(t2v_vae* v, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out);
/* z [B, z_channels, F, h, w] fp32/fp16 latent as returned by the sampler; multiplied by `z_scale`
 * (1/0.18215, t2v_pipeline.py:348) on ingest.
 *   out_mode 0: float32 [B*F, 3, 8h, 8w] in [-1, 1]   (what AutoencoderKL.decode returns, per frame)
 *   out_mode 1: uint8   [B*F, 8h, 8w, 3] RGB, tensor2vid arithmetic (t2v_pipeline.py:447-460)          */
int t2v_vae_decode(t2v_vae* v, const void* z, int z_is_f32, float z_scale, void* out, int out_mode, int B, int F, int h,
                   int w, void* stream);
/* moments = quant_conv(Encoder(x)) of AutoencoderKL.encode (modelscope/t2v_model.py:1640-1644; ldm Encoder ≙
 * videocrafter/lvdm/models/modules/autoencoder_modules.py:382-482): x [N, 3, H, W] fp16/fp32 in [-1, 1] (device) ->
 * moments_out [N, 2*embed_dim, H/8, W/8] fp32 = (mean | logvar).  compute_latents (t2v_pipeline.py:148-194) keeps
 * mean * 0.18215.  Needs the `encoder.*` / `quant_conv.*` parameters (optional for decode-only use). */
int t2v_vae_encode(t2v_vae* v, const void* x, int x_is_f32, void* moments_out, int N, int H, int W, void* stream);
double t2v_vae_flops(t2v_vae* v, int nframes, int h, int w);
/* Frame chunking of long / high-resolution clips.  A plan's activation arena grows linearly with its frame count (0.83 GB per
 * 576 x 1024 decoded frame).  t2v_vae_decode / t2v_vae_encode run the whole clip as one plan when that plan is cached or
 * fits the memory budget -- exactly as without chunking -- and otherwise as ceil(frames / n) consecutive frame ranges
 * (in (b f) order, a range may cross a sample boundary), n the largest frame count whose plan fits, the last range the
 * tail; each range is written straight to its place in the caller's output.  A chunked call drops that direction's cached
 * plans before it starts and after it ends (synchronising the stream): chunk plans are sized to the free memory and would
 * otherwise starve the next network's plan.  Every op is per frame; only reduction
 * orders that depend on the frame count (GroupNorm grid, GEMM split-K) can move the last bits (DESIGN.md section 2).
 * If even one frame does not fit, the call fails (-4) before allocating anything.
 *   direction: 0 = decode, 1 = encode; h, w as the entry point takes them (latent for decode, image for encode).
 *   plan_bytes: arena and GroupNorm workspace bytes a plan of this shape would allocate (host only, no GPU needed).
 *   plan_chunks: the split the policy picks for `budget` bytes (host only); -4 if one frame does not fit.
 *   set / get_memory_budget: bytes of plan (arena + GroupNorm workspace) one direction may hold; 0 (default) = automatic:
 *     free device memory + this direction's cached arenas + the GroupNorm workspace - 512 MB.
 *   last_chunking: how the last call of that direction was split (n_chunks = 1: the whole-clip plan; 0 before any call).
 *   cached_plans: number of cached plans of that direction and (if non-null) their arena bytes together.            */
int t2v_vae_plan_bytes(t2v_vae* v, int direction, int frames, int h, int w, size_t* arena, size_t* gn_workspace);
int t2v_vae_plan_chunks(t2v_vae* v, int direction, int frames, int h, int w, size_t budget, int* chunk_frames, int* n_chunks);
int t2v_vae_set_memory_budget(t2v_vae* v, size_t bytes);
size_t t2v_vae_get_memory_budget(t2v_vae* v);
int t2v_vae_last_chunking(t2v_vae* v, int direction, int* chunk_frames, int* n_chunks);
int t2v_vae_cached_plans(t2v_vae* v, int direction, size_t* slab_bytes);
/* Block outputs for parity tests.  enable_taps drops both directions' cached plans; plans built while taps are on keep the
 * output of every block under the reference module's name and never reuse its bytes (a larger arena; plan_bytes counts
 * it).  Decoder: "decoder.conv_in", "decoder.mid.block_1", "decoder.mid.attn_1", "decoder.mid.block_2", "decoder.up.<lvl>"
 * (after the level's upsample conv, if any), "decoder.norm_out" (GroupNorm + swish).  Encoder: "encoder.conv_in",
 * "encoder.down.<lvl>" (after the level's downsample conv, if any), "encoder.mid.block_1", "encoder.mid.attn_1",
 * "encoder.mid.block_2", "encoder.norm_out".  tap_info / read_tap read the most
 * recent plan of the tap's direction (a chunked call keeps none): rows x C tokens of frames of h x w, read as fp16
 * [rows / (h w), C, h, w].  read_tap returns the element count, or < 0 with the error set.                          */
int t2v_vae_enable_taps(t2v_vae* v, int on, void* stream);
int t2v_vae_tap_info(t2v_vae* v, const char* name, long long* rows, int* C, int* h, int* w);
long long t2v_vae_read_tap(t2v_vae* v, const char* name, void* dst, long long cap_elems, void* stream);
/* VideoCrafter LoRA on the decoder's and the encoder's weights (see "VideoCrafter LoRA" above) */
int t2v_vae_lora_apply(t2v_vae* v, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                       void* stream);
int t2v_vae_lora_restore(t2v_vae* v, const char* weight_name, void* stream);
int t2v_vae_lora_clear(t2v_vae* v, void* stream);
int t2v_vae_lora_merged(t2v_vae* v);

/* ------------------------------------------------------------------------------------------ text conditioning
 * replaces FrozenOpenCLIPEmbedder.encode_with_transformer (modelscope/clip_hardcode.py:112-119, :269-274): the OpenCLIP
 * ViT-H-14 text transformer (token + positional embedding, `layers_run` residual attention blocks with the causal mask --
 * 23 of the 24 for layer = 'penultimate' -- then ln_final; no text projection).  Parameter names are open_clip's
 * (`token_embedding.weight`, `positional_embedding`, `transformer.resblocks.N.{ln_1,attn.in_proj_weight,attn.in_proj_bias,
 * attn.out_proj,ln_2,mlp.c_fc,mlp.c_proj}`, `ln_final`), i.e. the keys of open_clip_pytorch_model.bin without `visual.*`.
 * Prompt parsing / chunking / emphasis weights stay host Python (clip_hardcode.py:146-395).
 * arch = 1 is VideoCrafter's FrozenCLIPEmbedder (videocrafter/lvdm/models/modules/condition_modules.py:15-40): the
 * OpenAI CLIP ViT-L/14 text model as transformers' CLIPTextModel computes `last_hidden_state` (all layers, then
 * final_layer_norm; quick_gelu MLP; causal mask only, no padding mask).                                          */
typedef struct t2v_clip t2v_clip;
typedef struct {
    int width;          /* 1024 (arch 1: 768) */
    int heads;          /* 16 (head width must be 64; arch 1: 12) */
    int layers_run;     /* 23 = 24 resblocks, 'penultimate' (arch 1: 12, every layer) */
    int context;        /* 77 */
    int vocab;          /* 49408 */
    int arch;           /* 0: OpenCLIP ViT-H-14 text tower, names above
                         * 1: transformers CLIPTextModel (ViT-L/14), state_dict keys relative to the CLIPTextModel:
                         *    `text_model.embeddings.{token_embedding,position_embedding}.weight`,
                         *    `text_model.encoder.layers.N.{layer_norm1,self_attn.{q,k,v,out}_proj,layer_norm2,mlp.fc1,
                         *    mlp.fc2}.{weight,bias}`, `text_model.final_layer_norm.{weight,bias}`; q / k / v are fused into
                         *    one projection inside the library.  A zero-initialised config is arch 0. */
} t2v_clip_config;
int t2v_clip_create(const t2v_clip_config* cfg, t2v_clip** out);
void t2v_clip_destroy(t2v_clip* m);
int t2v_clip_set_param(t2v_clip* m, const char* name, const void* data, int dtype, int ndim, const int64_t* shape, void* stream);
int t2v_clip_param_info(t2v_clip* m, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out);
/* tokens [B, context] int32 (device) -> out [B, context, width] fp16 (out_is_f32 = 0) or fp32: ln_final(transformer(...))
 * (arch 1: final_layer_norm(encoder(...)) = last_hidden_state) */
int t2v_clip_encode(t2v_clip* m, const int* tokens, void* out, int out_is_f32, int B, void* stream);
/* VideoCrafter LoRA on the tower's weights (see "VideoCrafter LoRA" above) */
int t2v_clip_lora_apply(t2v_clip* m, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                        void* stream);
int t2v_clip_lora_restore(t2v_clip* m, const char* weight_name, void* stream);
int t2v_clip_lora_clear(t2v_clip* m, void* stream);
int t2v_clip_lora_merged(t2v_clip* m);

/* ------------------------------------------------------------------------------------------ depth adapter
 * replaces VideoCrafter's T2I-Adapter (videocrafter/lvdm/models/modules/adapter.py: Adapter(channels, nums_rb, cin, ksize, sk,
 * use_conv)) as T2VAdapterDepth.get_adapter_features runs it (videocrafter/lvdm/models/ddpm3d.py:1470-1484): PixelUnshuffle(8),
 * conv_in, then nums_rb ResnetBlocks per level (the first block of every level after the first downsamples: 3x3 stride-2
 * conv if use_conv, else 2x2 average pooling), one feature map per level.  Parameter names are the reference module's
 * (`conv_in.*`, `body.{k}.{in_conv,block1,block2,skep,down_opt.op}.*`, k = level * nums_rb + block), so an adapter
 * checkpoint loads as is.  create rejects what the reference cannot run: sk = 0 with differing level widths (its skep is
 * built for the block's input width but applied to in_conv's output).  Also rejected: cin not a multiple of 64, ksize other
 * than 1 or 3, level widths not multiples of 8.                                                                      */
typedef struct t2v_adapter t2v_adapter;
typedef struct {
    int cin;              /* input channels after PixelUnshuffle(8): 64 * condition channels (64 for one depth channel) */
    int channels[4];      /* per-level widths, e.g. 320, 640, 1280, 1280 */
    int n_levels;         /* len(channels), 1..4 */
    int nums_rb;          /* ResnetBlocks per level */
    int ksize;            /* in_conv / block2 / skep kernel (1 or 3); block1 is always 3x3 */
    int sk;               /* 1: identity skip (in_conv only where the width changes), 0: skep conv in every block */
    int use_conv;         /* downsampling: 1 = 3x3 stride-2 conv (sizes round up), 0 = 2x2 average pooling (sizes round down) */
} t2v_adapter_config;
int t2v_adapter_create(const t2v_adapter_config* cfg, t2v_adapter** out);
void t2v_adapter_destroy(t2v_adapter* a);
int t2v_adapter_set_param(t2v_adapter* a, const char* name, const void* data, int dtype, int ndim, const int64_t* shape,
                          void* stream);
int t2v_adapter_missing_params(t2v_adapter* a, char* name_out, size_t name_cap);
int t2v_adapter_param_info(t2v_adapter* a, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out);
/* cond [N, cin/64, H, W] fp32 (cond_is_f32 = 1) or fp16 -> feats_out[i] [N, h_i, w_i, channels[i]] fp16 channels-last (the
 * reference's feature i [N, C_i, h_i, w_i], permuted), h_0 = H/8 and each later level halved as the config downsamples.
 * Errors: H or W not a multiple of 8, or a level that would be empty.  The first call at a shape builds its plan, the
 * second and later ones replay it as one CUDA graph.                                                                */
int t2v_adapter_encode(t2v_adapter* a, const void* cond, int cond_is_f32, void* const* feats_out, int N, int H, int W,
                       void* stream);
/* VideoCrafter LoRA on the adapter's weights (see "VideoCrafter LoRA" above) */
int t2v_adapter_lora_apply(t2v_adapter* a, const char* weight_name, const void* up, const void* down, int dtype, int rank,
                           float alpha, void* stream);
int t2v_adapter_lora_restore(t2v_adapter* a, const char* weight_name, void* stream);
int t2v_adapter_lora_clear(t2v_adapter* a, void* stream);
int t2v_adapter_lora_merged(t2v_adapter* a);

/* ------------------------------------------------------------------------------------------ sampler steps
 * replace the per-step tensor arithmetic of scripts/samplers (ddim/gaussian_sampler.py:125-136,:269-283;
 * ddim/sampler.py:176-218; uni_pc/uni_pc.py:299-307,:378-391,:625-650).                                  */
int t2v_ddim_step(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x_out, long long n,
                  long long chan_stride,
                  int C, int guided_channels, float g, int mode, float a0, float a1, float a2, float a3, float a4,
                  const float* noise, int cfg_fp16, void* stream);
/* t2v_ddim_step with VideoCrafter's per-step outputs (videocrafter/lvdm/samplers/ddim.py:230-279):
 *   cfg_variant  the guidance formula on the guided channels, fp32 op by op as torch evaluates it (uc_type):
 *                0 u + g (c - u) (None; the formula of t2v_ddim_step, fp16 rounding when cfg_fp16), 1 c + g (c - u)
 *                ('cfg_original'), 2 c + g (u - c) ('cfg_ours').  Variants 1 and 2 need cfg_fp16 = 0.  Without eps_u no
 *                guidance runs, whatever the variant.
 *   x0_out       NULL, or n fp32 elements that receive pred_x0 = (x - a0 e) / a1, the exact value the update then uses;
 *                mode 1 only.  The same pass writes it: one extra 4-byte store per element.
 * Variant 0 with x0_out = NULL launches the kernel t2v_ddim_step launches, so its output is bit-identical.  Errors (-1, before
 * any launch): cfg_variant outside 0..2, a variant 1 or 2 with cfg_fp16, x0_out with mode != 1, and x0_out overlapping x,
 * x_out, eps_c, eps_u or noise.                                                                                            */
int t2v_ddim_step_ex(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x_out, long long n,
                     long long chan_stride, int C, int guided_channels, float g, int mode, float a0, float a1, float a2, float a3,
                     float a4, const float* noise, int cfg_fp16, int cfg_variant, float* x0_out, void* stream);
int t2v_cfg_x0(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x0, long long n, float g,
               float alpha, float sigma, int cfg_fp16, void* stream);
int t2v_lincomb(float* out, const float* const* src, const float* coef, int n_src, long long n, void* stream);

/* x0 range restriction of DDIM_Gaussian (gaussian_sampler.py:110-120, :174-178, :199-202): t2v_ddim_step's mode 0 over B
 * samples of n / B elements each, with x0 restricted before eps is recomputed from it.
 *   percentile in (0, 1]: dynamic thresholding, per sample: s = the percentile-quantile of |x0| (as t2v_abs_quantile, written
 *                         to s_out [B]), then x0 = min(s', max(-s', x0)) / s' with s' = max(s, 1);
 *   percentile == 0:      x0 clamped to [-1, 1] (the reference clamps to +-1 whatever value `clamp` has); s_out and the
 *                         workspace are unused and may be NULL.
 * fp32 op by op in the reference's order; NaN propagates as in torch.  x_out holds x0 between the launches, so it must not
 * overlap x, eps_c, eps_u or noise.  Errors (-1, before any launch): x_out == x, n not a multiple of B, percentile outside
 * {0} U (0, 1], and with percentile > 0 the t2v_abs_quantile errors for n / B.  No host synchronisation: graph-capturable. */
int t2v_ddim_step_threshold(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x_out, long long n,
                            long long chan_stride, int C, int guided_channels, float g, float a0, float a1, float a2, float a3,
                            float a4, const float* noise, int cfg_fp16, int B, float percentile, float* s_out, void* workspace,
                            long long workspace_bytes, void* stream);
/* out[b] = torch.quantile(|x[b*n : (b+1)*n]|, q) (linear interpolation) for b < B, bit for bit: rank = fp32(q) * (n - 1) in
 * fp32, the floor(rank)-th and ceil(rank)-th order statistics by an exact radix select on the bit patterns, then torch.lerp's
 * fp32 arithmetic with weight rank - floor(rank); NaN for a sample that holds a NaN.  x and out are device pointers; the
 * workspace holds at least t2v_abs_quantile_workspace(B) bytes of device memory and is cleared on the stream by each call.
 * Deterministic, no host synchronisation (graph-capturable).  Errors (-1, before any launch): B outside [1, 65535], n < 1,
 * q outside [0, 1], a missing pointer or a short workspace, and n > 2^24 ("quantile() input tensor is too large", as torch). */
int t2v_abs_quantile(const float* x, int B, long long n, float q, float* out, void* workspace, long long workspace_bytes,
                     void* stream);
/* Host only: the workspace bytes t2v_abs_quantile and t2v_ddim_step_threshold need for B samples. */
long long t2v_abs_quantile_workspace(int B);

/* img2vid inpainting latent of process_modelscope.py:170-219: masked_latents = image_latents * (1 - mask) + latent_noise * mask
 * with mask[:, :, f] = weights[f] (the per-frame schedule of T2VAnimKeys), evaluated in fp64 like the reference's numpy code.
 *   image_latents [BC, image_frames, hw] fp32 (image_frames = 1: one encoded image shared by all frames, or F)
 *   noise, out, mask_out [BC, F, hw] fp64 (mask_out may be NULL); weights [F] fp64 -- all device pointers            */
int t2v_latent_blend(const float* image_latents, int image_frames, const double* noise, const double* weights, double* out,
                     double* mask_out, int BC, int F, long long hw, void* stream);

/* VideoCrafter q_sample (videocrafter/lvdm/models/ddpm3d.py:283-286) and the masked-DDIM blend (lvdm/samplers/ddim.py:188-195)
 * over a fp32 latent of shape[5] = [B, C, T, h, w], with torch's fp32 rounding op by op (bit-identical to torch's ops):
 *   known = a[b] * x0 + s[b] * noise
 *   out   = known                                  (mask = img = NULL: q_sample)
 *   out   = known * mask + (1 - mask) * img        (blend)
 * a / s [B]: sqrt_alphas_cumprod[t_b] / sqrt_one_minus_alphas_cumprod[t_b].  x0, noise and mask are addressed through five
 * element strides each, 0 on a broadcast dimension (a frame mask [1,1,T,1,1], a region mask [1,1,1,h,w], a batch-1 x0);
 * img and out are contiguous and out may equal img.  All pointers are device pointers.  Errors: a dimension < 1, a negative
 * stride, a missing pointer, or exactly one of mask / img given.                                                     */
int t2v_q_sample_blend(const float* x0, const long long* x0_strides, const float* noise, const long long* noise_strides,
                       const float* a, const float* s, const float* mask, const long long* mask_strides, const float* img,
                       float* out, const int* shape, void* stream);

/* vid2vid / img2vid frame preparation (process_modelscope.py:115-137, :172-190): PIL's Image.resize((W, H), Image.LANCZOS)
 * of n uint8 RGB frames src [n, H0, W0, 3], then the reference's normalisation, as numpy and torch round it op by op:
 * (float32(x) / 255) * 2 - 1.  out [n, 3, H, W] is fp32, or fp16 (round to nearest of that fp32 value) when out_fp16.
 * Bit-identical to Pillow: a horizontal pass over the rows the vertical pass reads into tmp, a uint8 buffer of at least
 * n * H0 * W * 3 bytes (tmp_bytes; unused and may be NULL when W == W0), then the vertical pass; a size that does not
 * change skips its pass.  src, out and tmp are device pointers.  The coefficient tables are built on the host once per
 * (in, out) size pair and kept on the device.  Returns -1 without launching when n < 1, a size lies outside [1, 32768],
 * src or out is NULL, out is not aligned to its element size, or tmp is missing or too small. */
int t2v_frames_resize(const void* src, int n, int H0, int W0, void* out, int H, int W, int out_fp16, void* tmp,
                      long long tmp_bytes, void* stream);
/* Host only: those tables for in_size -> out_size pixels.  *ksize = taps per output pixel: 2 * ceil(3 * max(in / out, 1)) + 1,
 * or 1 when in == out (the identity, for the pass Pillow skips).  bounds [out_size][2] = (first input pixel, taps used);
 * coeffs [out_size][*ksize] = int32 weights with 22 fractional bits, 0 past the taps used.  bounds and coeffs may be NULL
 * (query *ksize first).  Returns -1 when a size lies outside [1, 32768] or ksize is NULL. */
int t2v_resize_coeffs(int in_size, int out_size, int* ksize, int* bounds, int* coeffs);

/* ------------------------------------------------------------------------------------------ kernel-level entry
 * points (used by the parity tests; the model-level calls above are built from exactly these launchers).   */
int t2v_op_gemm(const void* a, long long lda, int K, int nd, const int* dims, int ntaps, const int* tap_off,
                const void* w_packed, int n_alloc, int N, int b_batch_dim, int flags, void* out, long long ldo,
                const void* bias, int bias_rows, long long bias_stride, const void* residual, long long ldr,
                float alpha, int force_bn, int force_cg, void* stream);
/* t2v_op_gemm's problem through split-K, the path the model takes for contractions too small to fill the GPU: `splits`
 * splits are requested, *splits_used returns how many run (no split is left empty), each writes an fp32 partial into
 * scratch [splits_used][rows][N] (scratch_elems = its capacity), and a fix-up pass adds them in split order plus bias
 * (per sample with bias_rows) and residual.  Errors, before any launch: GEGLU, fp32 output, batched B, alpha != 1,
 * N % 8 != 0, output / residual / bias rows not 16-byte aligned, scratch too small. */
int t2v_op_gemm_splitk(const void* a, long long lda, int K, int nd, const int* dims, int ntaps, const int* tap_off,
                       const void* w_packed, int n_alloc, int N, int b_batch_dim, int flags, void* out, long long ldo,
                       const void* bias, int bias_rows, long long bias_stride, const void* residual, long long ldr,
                       float alpha, int splits, float* scratch, long long scratch_elems, int* splits_used, int force_bn,
                       int force_cg, void* stream);
/* Linear(LayerNorm(x)) with the LayerNorm folded into the GEMM, as the transformer blocks and text towers run it (eps 1e-5):
 * w_folded [N, K] = fp16(w * gamma), colsum [N] = sum_k w_folded, bias32 [N] = w @ beta + bias (fp32), rowstat [rows][2] =
 * (mean, rstd) of each x row; then out = rstd * (x @ w_folded^T - mean * colsum) + bias32 (+ residual).  The caller owns the
 * four intermediates.  w / bias are already GEGLU-packed when flags = GEMM_GEGLU (out then has N / 2 columns); flags is 0
 * or GEMM_GEGLU.  x rows: K % 8 == 0, K <= 2048. */
int t2v_op_ln_linear(const void* x, long long ldx, long long rows, int K, const void* w, const void* bias, const void* gamma,
                     const void* beta, int N, int flags, void* w_folded, float* colsum, float* bias32, float* rowstat,
                     const void* residual, long long ldr, void* out, long long ldo, int force_bn, int force_cg, void* stream);
int t2v_op_pack_conv_weight(const void* src, int src_is_f32, void* dst, int Cout, int Cin, int taps, int n_alloc,
                            int k_alloc, void* stream);
int t2v_op_pack_geglu_weight(const void* w, const void* b, int src_is_f32, void* wdst, void* bdst, int H, int K, int bn,
                             void* stream);
/* The LoRA merge kernels of t2v_unet_lora_merge and t2v_*_lora_apply on a plain fp16 buffer w [out, cols] (the first
 * out * cols elements are written, nothing past them):
 *   t2v_op_lora_merge  w = fp16(w + fp16(fp16(B @ A) * alpha)), B [out, rank], A [rank, cols] fp16 (A [rank, 3 * cols] with
 *                      temporal_mean: the product viewed [out, cols / 3, 3, 3] and averaged over its last axis);
 *   t2v_op_lora_apply  w = fp16(w + alpha * up @ down) in fp32, up [out, rank], down [rank, cols], fp16 (dtype 0) or fp32
 *                      (dtype 1).
 * All pointers are device pointers.  Errors (-1, before any launch): rank, out or cols < 1, dtype other than 0 or 1. */
int t2v_op_lora_merge(void* w, const void* A, const void* B, int out, int cols, int rank, float alpha, int temporal_mean,
                      void* stream);
int t2v_op_lora_apply(void* w, const void* up, const void* down, int dtype, int out, int cols, int rank, float alpha,
                      void* stream);
/* GroupNorm (32 groups, + SiLU when silu) of instances of rows_per_inst consecutive rows of x [rows, C] -> y.
 * phase 0: what the model runs on one GPU (one fused launch where the grid can be co-resident, else statistics + apply).
 * phase 1: statistics only, with the chunking of the frame-sharded plans; (mean, rstd) per (instance, group) go to
 *          stats, fp32 [rows / rows_per_inst, 32, 2].  y is not written.
 * phase 2: apply only, with the caller's stats in the same layout.
 * Returns -1 without launching on bad arguments: C not a positive multiple of 32 up to 2560, rows not 1 to 65535 whole
 * instances, x / y / gamma / beta not 16-byte aligned, ldx / ldy not multiples of 8 or below C; -5 if the workspace cannot
 * be allocated. */
int t2v_op_groupnorm(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, int rows_per_inst,
                     const void* gamma, const void* beta, float eps, int silu, int phase, float* stats, void* stream);
/* LayerNorm over C of every row.  Returns -1 without launching unless C % 8 == 0, 8 <= C <= 2048, 1 <= rows < 2^31, x / y /
 * gamma / beta are 16-byte aligned and ldx, ldy are multiples of 8 and >= C. */
int t2v_op_layernorm(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, const void* gamma,
                     const void* beta, float eps, void* stream);
/* softmax(Q K^T * scale) V, head_dim 64, head h at column h * 64; batch b reads Q / O at b * X_bs and K / V at
 * (b / kv_batch_div) * X_bs.  Strides in elements.  Returns -1 without launching on operands the kernels cannot load:
 * Q, K, V not 16-byte aligned or a Q / K / V stride not a multiple of 8 (0 is allowed), O not 4-byte aligned or an odd
 * O stride. */
int t2v_op_attention(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_ss,
                     long long k_bs, long long k_ss, long long v_bs, long long v_ss, long long o_bs, long long o_ss,
                     int batch, int heads, int sq, int skv, int kv_batch_div, float scale, void* stream);
/* same for head_dim in {8,16,32,40,80,160} (64 dispatches to t2v_op_attention's kernels): CrossAttention.forward of the
 * VideoCrafter denoiser, videocrafter/lvdm/models/modules/attention_temporal.py:167-190 (8 heads of width C/8), plus a
 * two-level batch: batch index b -> (b / b_inner) * X_bs + (b % b_inner) * X_bsi for X in q, k, v, o (K / V after the
 * kv_batch_div division); b_inner = 1 leaves the X_bsi unused.  With head_dim 64 this reaches the ModelScope temporal
 * attention layout (outer = sample, inner = pixel, sequence = frames).  Same alignment rules as t2v_op_attention. */
int t2v_op_attention_hd(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_ss,
                        long long k_bs, long long k_ss, long long v_bs, long long v_ss, long long o_bs, long long o_ss,
                        int batch, int heads, int head_dim, int sq, int skv, int kv_batch_div, float scale, int b_inner,
                        long long q_bsi, long long k_bsi, long long v_bsi, long long o_bsi, void* stream);
/* TemporalCrossAttention.forward with RelativePosition tables (attention_temporal.py:46-65, :107-144), context = x:
 * sequences of T <= 32 frames; sequence s of n_seq lives at (s / seq_inner) * bs_outer + (s % seq_inner) * bs_inner, its
 * frames `ss` elements apart; head h at column h * head_dim; tables [2*max_rel+1, head_dim] fp16 (2*max_rel+1 <= 48),
 * frame distances beyond +-max_rel use the end rows of the tables, as the reference's clamp.  Same alignment rules as
 * t2v_op_attention, and the tables 16-byte aligned. */
int t2v_op_attention_relpos(const void* q, const void* k, const void* v, void* o, const void* table_k, const void* table_v,
                            long long n_seq, long long seq_inner, long long bs_outer, long long bs_inner, long long ss,
                            long long o_bs_outer, long long o_bs_inner, long long o_ss, int heads, int head_dim, int T,
                            int max_rel, float scale, void* stream);
/* The CLIP / OpenCLIP text towers' causal self-attention (nn.MultiheadAttention with the causal mask): qkv [B*L, 3W] fp16
 * as in_proj lays it out (q | k | v, head h at columns h*64 of each part) -> o [B*L, W]; q is scaled by 64^-0.5 before
 * q.k as nn.MultiheadAttention does.  -1 unless W % 64 == 0, W / heads == 64 and 1 <= L <= 128. */
int t2v_op_clip_attention(const void* qkv, void* o, int B, int L, int W, int heads, void* stream);
int t2v_op_upsample2x(const void* x, void* y, int nframes, int h, int w, int C, void* stream);
/* 3x3 stride-2 gather x [n, h, w, C] -> col [n*ho*wo, 9*C] (tap-major, tap = ky*3+kx), zeros outside x.  pad_lo = 1:
 * Conv2d(stride 2, padding 1), ho = ceil(h/2); pad_lo = 0: the ldm Downsample's pad (0,1,0,1) + padding 0, ho = floor(h/2).
 * -1 unless C % 8 == 0 and pad_lo is 0 or 1. */
int t2v_op_im2col_s2(const void* x, void* col, int nframes, int h, int w, int C, int pad_lo, void* stream);
int t2v_op_time_sinusoid(const float* t, void* out, int B, int dim, void* stream);
int t2v_op_small_linear(const void* x, long long ldx, const void* W, const void* bias, const void* addend, void* y,
                        long long ldy, int B, int N, int K, int silu_in, void* stream);
/* Frames [frame0, frame0 + nframes) in (b f) order of x [B, C, F, h, w] (fp32 or fp16) -> tok [nframes*h*w, ld] fp16:
 * column c < C = fp16(x * scale) (fp32 product, one rounding), columns C..cpad-1 = 0, columns >= cpad untouched. */
int t2v_op_ingest_latent(const void* x, int x_is_f32, void* tok, long long ld, int cpad, int C, int F, int h, int w,
                         long long frame0, long long nframes, float scale, void* stream);
/* tok [B*F*h*w, ld] fp16 (columns 0..C-1) -> out [B, C, F, h, w] fp32 (exact) or fp16 (copied). */
int t2v_op_egress_latent(const void* tok, long long ld, void* out, int out_is_f32, int B, int C, int F, int h, int w,
                         void* stream);
/* nn.AvgPool2d(2, 2) of x [n, h, w, C] -> y [n, h/2, w/2, C] (floor sizes): fp32 sum of the four taps in row-major order,
 * times 0.25, one fp16 rounding.  -1 unless C % 8 == 0. */
int t2v_op_avgpool2x2(const void* x, void* y, int nframes, int h, int w, int C, void* stream);
/* nn.PixelUnshuffle(8) of x [N, Cc, H, W] (fp32 rounded once, or fp16) -> tok [N*(H/8)*(W/8), 64*Cc] fp16.
 * -1 unless H % 8 == 0 and W % 8 == 0. */
int t2v_op_pixel_unshuffle(const void* x, int x_is_f32, void* tok, int N, int Cc, int H, int W, void* stream);
/* nn.ReLU in place on a dense fp16 matrix [rows, C]; NaN stays NaN.  -1 unless C % 8 == 0. */
int t2v_op_relu(void* x, long long rows, int C, void* stream);
/* x[r, :C] = fp16(x[r, :C] + f[(s % f_samples) * rows_per_sample + r % rows_per_sample, :]) with s = r / rows_per_sample, f dense
 * [., C]; fp32 add, one rounding.  -1 unless C and ldx are multiples of 8 and rows_per_sample, f_samples >= 1. */
int t2v_op_feature_add(void* x, long long ldx, const void* f, int C, long long rows, long long rows_per_sample, int f_samples,
                       void* stream);
/* out[r, :Ca + Cb] = a[r, :Ca] | b[r, :Cb], copied.  -1 unless Ca, Cb, lda, ldb and ldo are multiples of 8. */
int t2v_op_concat_cols(const void* a, long long lda, int Ca, const void* b, long long ldb, int Cb, void* out, long long ldo,
                       long long rows, void* stream);
/* y = softmax over each dense row of x [rows, cols] of fp16(x * scale): fp32 math with __expf, one output rounding. */
int t2v_op_softmax_rows(const void* x, void* y, long long rows, int cols, float scale, void* stream);
/* x [nb, R, C] -> y [nb, C, R] fp16, copied. */
int t2v_op_transpose_batched(const void* x, void* y, int nb, int R, int C, void* stream);
/* tok [pixels, ld] fp16, RGB in columns 0..2 -> out [pixels, 3] uint8 = trunc(clamp(v * 0.5 + 0.5, 0, 1) * 255) in fp32; NaN -> 0. */
int t2v_op_frames_to_u8(const void* tok, long long ld, void* out, long long pixels, void* stream);
/* tok [n*H*W, ld] fp16, RGB in columns 0..2 -> out [n, 3, H, W] fp32 (exact). */
int t2v_op_frames_to_f32(const void* tok, long long ld, float* out, int n, int H, int W, void* stream);
/* dst [n] fp16 = src (fp32 rounded to nearest even, or fp16 copied). */
int t2v_op_convert_to_f16(const void* src, int src_is_f32, void* dst, long long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* T2V_B200_H */

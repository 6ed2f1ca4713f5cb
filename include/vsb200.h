/* libvsb200.so — C ABI of the H100-native (sm_90a) VideoSeal embed/detect hot path.
 *
 * Plain pointers and sizes only (no torch types).  All `*_dev` pointers are CUDA device pointers on the
 * device the model was finalised on; `stream` is a cudaStream_t passed as void*.  Every entry point returns
 * 0 on success or a negative vsb_status; vsb_last_error() gives the message.  There is NO CPU fallback:
 * on any device other than compute capability 9.0 (H100) vsb_model_finalize() fails.
 *
 * Each entry point names the reference interface it replaces (paths relative to facebookresearch/videoseal):
 *   vsb_model_create / set_tensor / finalize  <-  videoseal/utils/cfg.py:88-149 setup_model (build_embedder
 *        models/embedder.py:243, build_extractor models/extractor.py:170, load_state_dict of checkpoint['model'])
 *   vsb_embed                                 <-  models/wam.py:134-204 Wam.embed and models/videoseal.py:258-350
 *        Videoseal.embed (resize, RGB->Y, UnetEmbedder.forward embedder.py:151, _apply_video_mode, JND.heatmaps
 *        modules/jnd.py:80, Blender.additive_blend blender.py:61, clamp)
 *   vsb_embedder_forward                      <-  models/embedder.py:151-165 UnetEmbedder.forward (operator seam)
 *   vsb_detect                                <-  models/wam.py:206-234 Wam.detect / videoseal.py:352-388 (resize,
 *        ConvnextExtractor.forward models/extractor.py:154, or SegmentationExtractor.forward models/extractor.py:55-69)
 *   vsb_jnd_heatmaps                          <-  modules/jnd.py:80-108 JND.heatmaps (operator seam)
 *   vsb_embed_host / vsb_detect_host          <-  the same calls with HOST (CPU) tensors as the reference keeps
 *        full-resolution video on the CPU (evals/full.py:117-120); H2D/D2H copies happen inside.
 */
#ifndef VSB200_H
#define VSB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vsb_model vsb_model;

enum vsb_status {
  VSB_OK = 0,
  VSB_ERR_INVALID = -1,      /* bad argument / shape */
  VSB_ERR_UNSUPPORTED = -2,  /* card feature outside the hot path (raise at load() time) */
  VSB_ERR_CUDA = -3,         /* CUDA error, message in vsb_last_error() */
  VSB_ERR_STATE = -4         /* call order (e.g. embed before finalize, missing weight) */
};

enum vsb_video_mode { VSB_VIDEO_REPEAT = 0, VSB_VIDEO_ALTERNATE = 1, VSB_VIDEO_INTERPOLATE = 2 };

/* Resizes follow the reference's `interpolation` dict, F.interpolate(size=..., **interpolation) at both resize sites (frames to
 * img_size, wam.py:161-164 / videoseal.py:305; the delta back to the frame size, wam.py:183-185 / videoseal.py:329).  The mode sits
 * in bits 5-6 (VSB_FLAG_RESIZE_MODE(m)); all resize bits zero = bilinear, align_corners=False, antialias=True.  Nearest and area
 * need VSB_FLAG_RESIZE_NO_AA and no VSB_FLAG_RESIZE_ALIGN_CORNERS (F.interpolate raises ValueError otherwise; here
 * VSB_ERR_INVALID when a resize happens).  Outputs of bicubic resizes are not clamped (only imgs_w is, by VSB_FLAG_CLAMP). */
enum vsb_resize_mode { VSB_RESIZE_BILINEAR = 0, VSB_RESIZE_BICUBIC = 1, VSB_RESIZE_NEAREST = 2, VSB_RESIZE_AREA = 3 };

enum vsb_flags {
  VSB_FLAG_CLAMP = 1,            /* clamp imgs_w to [0,1]           (wam.py:196-197) */
  VSB_FLAG_LOWRES_ATTN = 2,      /* JND at processing resolution    (wam.py:177-180) */
  VSB_FLAG_NO_ATTENUATION = 4,   /* model.attenuation = None        */
  VSB_FLAG_RESIZE_NO_AA = 8,     /* interpolation antialias=False   (videoseal.py:394) */
  VSB_FLAG_RESIZE_ALIGN_CORNERS = 16,   /* interpolation align_corners=True */
  VSB_FLAG_RESIZE_MODE_SHIFT = 5,       /* interpolation mode: a vsb_resize_mode in bits 5-6 */
  VSB_FLAG_RESIZE_MODE_MASK = 0x60
};
#define VSB_FLAG_RESIZE_MODE(m) ((int32_t)(m) << VSB_FLAG_RESIZE_MODE_SHIFT)
/* the bits of vsb_flags that describe a resize */
#define VSB_FLAG_RESIZE_BITS (VSB_FLAG_RESIZE_NO_AA | VSB_FLAG_RESIZE_ALIGN_CORNERS | VSB_FLAG_RESIZE_MODE_MASK)

/* Architecture hyper-parameters taken from the model card (videoseal/cards/<card>.yaml). */
typedef struct vsb_model_desc {
  int32_t nbits;             /* args.nbits */
  int32_t hidden;            /* int(nbits * hidden_size_multiplier), embedder.py:244 */
  int32_t img_size;          /* args.img_size_proc | img_size_extractor */
  int32_t yuv;               /* 'yuv' in embedder.model, embedder.py:281 */
  int32_t unet_in_ch, unet_out_ch;
  int32_t unet_levels;       /* len(z_channels_mults), <= 6 */
  int32_t unet_z[6];         /* z_channels * mult */
  int32_t unet_num_blocks;
  int32_t unet_act;          /* 0 relu (the only value the GPU path implements; 1 = silu is rejected by vsb_model_create) */
  int32_t unet_norm;         /* 0 batch (the only value the GPU path implements; 1 = rms is rejected by vsb_model_create) */
  int32_t unet_last_tanh;
  int32_t ext_depths[4];
  int32_t ext_dims[4];       /* after proportional_dim scaling, extractor.py:193-198 */
  int32_t ext_stem_stride;
  int32_t jnd_in_ch, jnd_out_ch; /* configs/attenuation.yaml entry (jnd_1_1 / jnd_1_3 / jnd_3_1 / jnd_3_3); 0,0 = no attenuation */
} vsb_model_desc;

const char* vsb_last_error(void);
int vsb_version(void);

/* Checks every rule on the descriptor and chooses each U-Net layer's kernel, with no CUDA call (a load-time dry run needs no GPU).
 * VSB_ERR_UNSUPPORTED unless: BatchNorm+ReLU; U-Net widths 16, 32, multiples of 64, or 8 in leading levels but not the last; up
 * blocks of 8 * 2^k <= 512 channels; img_size >> (levels - 1) >= 16; img_size <= 768 with 8 channels, whose layers must fit their
 * rings; JND channels 1 or 3.  VSB_ERR_INVALID unless: 2..6 levels, unet_in_ch 1 (yuv) or 3, unet_out_ch 1..3, img_size a multiple
 * of 128, hidden a multiple of 8, ConvNeXt widths even and not shrinking.  unet_levels 0 with unet_in_ch = unet_out_ch = 3
 * leaves the embedder to vsb_model_set_hidden_embedder; the U-Net rules are then checked at finalize if none was set. */
int vsb_model_create(const vsb_model_desc* desc, vsb_model** out);
/* Temporal U-Net (unet.conv_layer 'conv3d', modules/common.py Conv3dWrapper), called between create and finalize; no CUDA call.
 * on = 1: every ResnetBlock's 3x3 convs are 3x3x3 over the key frames of one embedder call (see vsb_embed) and its res_conv 1x1x1; the
 * checkpoint then holds their 5-D weights under the Conv3dWrapper keys (`...double_conv.0.conv.weight`).  on = 0: 'conv2d', the default.
 * VSB_ERR_UNSUPPORTED for a U-Net width below 16; VSB_ERR_STATE after finalize; VSB_ERR_INVALID for on other than 0 / 1. */
int vsb_model_set_unet_temporal(vsb_model* m, int32_t on);
/* one state_dict entry, fp32, host memory, contiguous, at most 5 dimensions; `name` is the reference state_dict key */
int vsb_model_set_tensor(vsb_model* m, const char* name, const float* data, const int64_t* shape, int32_t ndim);
/* Pixel-wise extractor head (modules/pixel_decoder.py:44-83 with pixelwise=True), called between create and finalize.  Without
 * this call the model has the pooled head (one [1+nbits] logit vector per frame).  pixelwise = 1 needs 1..8 stage factors, each 2
 * or 4, and a ConvNeXt trunk with ext_stem_stride 4 or a SAM-ViT trunk; stage i maps C -> C / factors[i] channels (bilinear up-sampling, reflect-padded
 * 3x3 conv, LayerNorm, GELU), then a 1x1 conv gives 1+nbits maps.  pixelwise = 0 accepts only n_stages = 1, factors = {1} (the
 * pooled head).  A SAM-ViT trunk (vsb_model_set_vit_extractor, called first) has width out_chans on an img_size / 16 map and no
 * stem-stride rule.  Like vsb_model_create it makes no CUDA call, and it returns VSB_ERR_UNSUPPORTED unless: the trunk width
 * (ext_dims[3] or out_chans) is 16, 32 or >= 64; every stage width C / f is a whole multiple of 8, of the form 8 * {1, 3} * 2^k (k <= 5) for a
 * middle stage and at most 32 for the last; the last stage's input map is a multiple of 16 / f pixels, and its staged taps,
 * (16 / f + 2)^2 * 9 * C fp16, plus its head weights, (1 + nbits) * (C + 1) fp32, fit in 227 KB.  VSB_ERR_STATE after finalize;
 * VSB_ERR_INVALID / VSB_ERR_UNSUPPORTED for other values. */
int vsb_model_set_pixel_decoder(vsb_model* m, int32_t n_stages, const int32_t* factors, int32_t pixelwise);
/* SAM-ViT extractor (models/extractor.py:41-69 SegmentationExtractor, modules/vit.py ImageEncoderViT with use_abs_pos), replacing the
 * ConvNeXt trunk; the ext_* fields of the model descriptor are then unused (zero).  The trunk's output is out_chans channels on a
 * grid = img_size / 16 map, which the pooled head or the pixel-wise decoder reads as it reads the ConvNeXt trunk's. */
typedef struct vsb_vit_desc {
  int32_t embed_dim, depth, num_heads, patch_size, window_size;
  uint32_t global_mask;      /* bit i set: block i attends over the whole grid (global_attn_indexes), else over windows */
  int32_t mlp_dim;           /* int(embed_dim * mlp_ratio) */
  int32_t out_chans;         /* neck width */
  int32_t qkv_bias, use_rel_pos;
} vsb_vit_desc;
/* Called after vsb_model_create and before vsb_model_set_pixel_decoder and finalize; no CUDA call.  VSB_ERR_STATE after finalize.
 * VSB_ERR_UNSUPPORTED unless: head dim embed_dim / num_heads = 64; mlp_dim and out_chans multiples of 64; patch_size 16; depth <= 32;
 * grid = img_size / 16 divisible by window_size (no window padding) and every window a multiple of 64 tokens (window 8 passes, 14
 * does not); global attention over at most 1024 tokens (img_size <= 512); with use_rel_pos, windows at most 32 tokens wide (the
 * 2n - 1 rows of a relative-position table must fit in 64).  VSB_ERR_INVALID for depth < 1, mask bits at or above
 * depth, or flags other than 0 / 1. */
int vsb_model_set_vit_extractor(vsb_model* m, const vsb_vit_desc* vit);
/* HiDDeN networks (modules/hidden.py HiddenEncoder / HiddenDecoder; models/embedder.py HiddenEmbedder, models/extractor.py
 * HiddenExtractor): stacks of ConvBNRelu = 3x3 conv (pad 1, bias) + norm + activation on x = 2 imgs - 1.
 *   embedder: num_layers ConvBNRelu (3 -> z, then z -> z), the concat [2 m - 1 as nbits constant planes | features | x], one
 *             ConvBNRelu (nbits + z + 3 -> z), final_layer 1x1 (z -> 3), tanh when last_tanh.  Its output is the delta (3 channels).
 *   extractor: num_layers ConvBNRelu (num_blocks + 1 of the reference), the mean over the map, Linear(z -> 1 + nbits): the pooled
 *             logits.
 * The embedder replaces the U-Net: the descriptor's unet_* fields are then unused (unet_levels 0, unet_in_ch = unet_out_ch = 3).  The extractor replaces the
 * trunk and the pixel decoder: ext_* zero, no vsb_model_set_vit_extractor, no pixel-wise vsb_model_set_pixel_decoder. */
typedef struct vsb_hidden_desc {
  int32_t z_channels;        /* width of every layer */
  int32_t num_layers;        /* ConvBNRelu layers before the concat (embedder) / before the pooling (extractor) */
  int32_t norm;              /* 0 BatchNorm2d (eval, eps 1e-5), 1 GroupNorm(8, z) (eps 1e-5, affine) */
  int32_t act;               /* 0 ReLU, 1 GELU (erf) */
  int32_t last_tanh;         /* embedder: tanh after final_layer; extractor: 0 */
} vsb_hidden_desc;
/* Called after vsb_model_create and before finalize; no CUDA call.  VSB_ERR_STATE after finalize (and for the extractor after a
 * SAM-ViT trunk or a pixel-wise decoder).  VSB_ERR_UNSUPPORTED unless z_channels is 64 and norm / act are 0 or 1.
 * VSB_ERR_INVALID for num_layers outside 1..64, last_tanh other than 0 / 1 (0 for the extractor), nbits < 1, img_size not a positive
 * multiple of 128, or a descriptor that does not leave room for it (unet_levels != 0 or RGB channels other than 3; ext_dims /
 * ext_depths != 0).  Such a descriptor with no HiDDeN embedder fails at finalize with the U-Net's VSB_ERR_INVALID. */
int vsb_model_set_hidden_embedder(vsb_model* m, const vsb_hidden_desc* h);
int vsb_model_set_hidden_extractor(vsb_model* m, const vsb_hidden_desc* h);
/* DVMark extractor (modules/dvmark.py DVMarkDecoder; models/extractor.py build_extractor 'dvmark'): 3x3x3 Conv3d over the frames of
 * one detector call, 3 -> 128 (ReLU), 128 -> 128 (ReLU), avgpool (1,2,2), 128 -> 256 (ReLU), avgpool (1,2,2), 256 -> 1 + nbits, the
 * mean over the map: pooled logits.  The frames are read in [0, 1] (no preprocess).  Checkpoint keys detector.layers.layer{1..4}.
 * {weight,bias}, 5-D weights.  It replaces the trunk and the pixel decoder like the HiDDeN extractor: ext_* zero, no
 * vsb_model_set_vit_extractor / vsb_model_set_hidden_extractor, no pixel-wise vsb_model_set_pixel_decoder (VSB_ERR_STATE /
 * VSB_ERR_INVALID / VSB_ERR_UNSUPPORTED).  Called after vsb_model_create and before finalize; no CUDA call.  VSB_ERR_INVALID for
 * nbits < 1 or nbits other than the descriptor's (any nbits >= 1 is implemented); VSB_ERR_UNSUPPORTED for an img_size that is not a
 * positive multiple of 128.  A group of frames convolved together is at most 64 long (vsb_detect_grouped). */
int vsb_model_set_dvmark_extractor(vsb_model* m, int32_t nbits);
/* DVMark embedder (modules/dvmark.py DVMarkEncoder; models/embedder.py DVMarkEmbedder, build_embedder 'dvmark'): Conv3d layers with
 * bias over the key frames of one embedder call on x = 2 imgs - 1, the message bits of each frame as nbits constant 0 / 1 planes:
 * (1,3,3) convs 3 -> 64 -> 64 -> 64 and a 3x3x3 64 -> 64 (ReLU); [x | planes] -> 256 -> 128 -> 128 (3x3x3, ReLU): x_skip;
 * [avgpool (1,2,2) of x_skip | planes] -> 512 -> 256 -> 256 (3x3x3, ReLU); bilinear up-sample (align_corners=True); [x_skip | up]
 * -> 256 -> 128 (3x3x3, ReLU) -> 3 (3x3x3), tanh: the delta (3 channels).  Checkpoint keys embedder.unet.{transform_layer.{0,2,4,6},
 * emb_layer{1,2,3}.{0,2,4}}.{weight,bias}, 5-D weights.  It replaces the U-Net like the HiDDeN embedder: unet_levels 0, unet_in_ch
 * = unet_out_ch = 3 (else VSB_ERR_INVALID).  Called after vsb_model_create and before finalize; no CUDA call.  VSB_ERR_STATE after
 * finalize or when the model already has a HiDDeN embedder or a temporal U-Net; VSB_ERR_INVALID for nbits < 1 or nbits other than
 * the descriptor's (any nbits >= 1 is implemented); VSB_ERR_UNSUPPORTED for an img_size that is not a positive multiple of 128 or
 * is above 512.  vsb_embed groups its key frames as for a temporal U-Net: at most 64 per group (chunk_keys). */
int vsb_model_set_dvmark_embedder(vsb_model* m, int32_t nbits);
/* VAE embedder (modules/vae.py VAEEncoder / VAEDecoder, modules/msg_processor.py 'binary+concat'; models/embedder.py VAEEmbedder,
 * build_embedder 'vae*'): decoder(msg_processor(encoder(2 imgs - 1), msgs)), 'yuv' cards on x = 2 Y - 1.  Levels of widths
 * ch * ch_mult[l] at S / 2^l; ResnetBlocks out = shortcut(x) + conv2(silu(GN2(conv1(silu(GN1(x)))))), GN = GroupNorm(16, C, eps 1e-6),
 * shortcut the identity or the 1x1 nin_shortcut; Downsample pad (0,1,0,1) + 3x3 stride 2; Upsample nearest x2 + 3x3; mid ResnetBlock,
 * single-head AttnBlock over the whole deepest grid (head dim = last width), ResnetBlock; encoder conv_out -> z_channels; the message
 * as hidden = nbits * hidden_size_multiplier constant planes sum_k E[2k + m_k] after the latent; decoder conv_out -> out_ch, tanh
 * when tanh_out: the delta (out_ch channels).  Checkpoint keys embedder.encoder.*, embedder.decoder.*,
 * embedder.msg_processor.msg_embeddings.weight.  It replaces the U-Net like the HiDDeN embedder: unet_levels 0, unet_in_ch =
 * unet_out_ch = 3 (else VSB_ERR_INVALID); its own channels travel in the descriptor. */
typedef struct vsb_vae_desc {
  int32_t in_ch;             /* encoder in_channels: 3, or 1 for the 'yuv' cards (then the descriptor's yuv is 1) */
  int32_t out_ch;            /* decoder out_ch: channels of the delta */
  int32_t ch;                /* base width */
  int32_t levels;            /* len(ch_mult), 1..6 */
  int32_t ch_mult[6];
  int32_t num_res_blocks;    /* encoder blocks per level (the decoder has num_res_blocks + 1) */
  int32_t z_channels;        /* encoder latent channels (double_z false) */
  int32_t tanh_out;          /* decoder tanh */
} vsb_vae_desc;
/* Called after vsb_model_create and before finalize; no CUDA call.  VSB_ERR_STATE after finalize or when the model already has a
 * HiDDeN, DVMark or temporal U-Net embedder.  VSB_ERR_INVALID for a descriptor that describes a U-Net, yuv != (in_ch == 1), in_ch
 * other than 1 / 3, levels outside 1..6, num_res_blocks outside 1..8, tanh_out other than 0 / 1 or non-positive widths.
 * VSB_ERR_UNSUPPORTED unless: every level width (and ch) is 16, 32, 64 or 128; the last-level width (the attention head dim) is 64
 * or 128; z_channels <= 16; out_ch 1 or 3; img_size a multiple of 128, at most 768, whose deepest map img_size / 2^(levels - 1)
 * is a whole multiple of 16 pixels and at most 96 (the attention's 9 216 tokens). */
int vsb_model_set_vae_embedder(vsb_model* m, const vsb_vae_desc* vae);
/* fold BN, pack to fp16 KRSC, upload to `device`, build nothing else (plans are built lazily per batch shape) */
int vsb_model_finalize(vsb_model* m, int32_t device);
void vsb_model_destroy(vsb_model* m);

/* imgs_dev [F,3,H,W] fp32 in [0,1]; msgs_dev uint8 {0,1}: [F,nbits] (n_msgs == F) or [1,nbits] (n_msgs == 1);
 * imgs_w_dev [F,3,H,W]; preds_w_dev NULL or [F,PC,H,W] (hmap * delta_up, before scaling_w; PC = max(unet_out_ch, jnd_out_ch) with
 * attenuation on, the broadcast of `hmaps * preds_w` in wam.py:189-193, else unet_out_ch);
 * step = 1 for image mode, else frames share the key frame f/step (videoseal.py:292-340);
 * chunk_keys = the model's chunk_size (key frames per reference chunk, videoseal.py:300): it only changes the result in
 * video_mode 'interpolate', where neighbouring key frames of ONE chunk are mixed (videoseal.py:101-113); 1..64 there.
 * A temporal U-Net (vsb_model_set_unet_temporal) convolves across the key frames of one group of chunk_keys consecutive key frames (one
 * reference embedder call: a video chunk, or, in image mode, the whole batch, so pass chunk_keys = F there); the last group may be
 * shorter, and frames of different groups never interact.  VSB_ERR_UNSUPPORTED when chunk_keys > 64 (a group must fit one
 * 64-frame sub-batch).  A DVMark embedder (vsb_model_set_dvmark_embedder) groups its key frames the same way.  The same holds for vsb_embed_host, vsb_embed_detect_host and vsb_frames_host_u8. */
int vsb_embed(vsb_model* m, const float* imgs_dev, const uint8_t* msgs_dev, int32_t n_msgs, float* imgs_w_dev,
              float* preds_w_dev, int32_t F, int32_t H, int32_t W, int32_t step, int32_t video_mode, int32_t chunk_keys,
              float scaling_i, float scaling_w, int32_t flags, void* stream);

/* x_dev [B, 3, S, S] RGB fp32 in [0,1] at processing size S = img_size (the Y extraction for yuv cards happens
 * inside, wam.py:168-172); delta_dev [B, unet_out_ch, S, S].  A temporal U-Net or a DVMark embedder takes the B frames as one group (one reference
 * embedder call): VSB_ERR_UNSUPPORTED for B > 64. */
int vsb_embedder_forward(vsb_model* m, const float* x_dev, const uint8_t* msgs_dev, int32_t n_msgs, float* delta_dev,
                         int32_t B, void* stream);

/* imgs_dev [F,3,H,W] -> logits_dev [F, 1+nbits]; for a pixel-wise model (vsb_model_set_pixel_decoder) logits_dev is
 * [F, 1+nbits, P, P] fp32 NCHW with P = (img_size / 32) * prod(factors), i.e. img_size for upscale_stages [4, 4, 2]:
 * channel 0 is the detection map, channels 1.. the per-pixel message bits (the reference's "b (1+nbits) h w").
 * The same shape applies to vsb_detect_host.  vsb_embed_detect_host and vsb_frames_host_u8 with logits_host != NULL
 * return VSB_ERR_UNSUPPORTED for pixel-wise models. */
int vsb_detect(vsb_model* m, const float* imgs_dev, float* logits_dev, int32_t F, int32_t H, int32_t W, int32_t flags,
               void* stream);
/* vsb_detect with the frames in groups of `group` consecutive frames (the last group may be shorter): one reference detector call
 * each, a video chunk of chunk_size frames (videoseal.py:373-379) or, in image mode, the whole batch (wam.py:206-234).  Only a DVMark
 * extractor convolves across the frames of a group; frames of different groups never interact, and the other extractors ignore
 * `group`.  DVMark: VSB_ERR_INVALID for group < 1, VSB_ERR_UNSUPPORTED for group > 64 (a group must fit one 64-frame sub-batch).
 * vsb_detect and vsb_detect_host take the whole call as one group (group = F).  vsb_embed_detect_host and vsb_frames_host_u8 with
 * logits_host != NULL, whose slices would split the groups, return VSB_ERR_UNSUPPORTED for a DVMark extractor. */
int vsb_detect_grouped(vsb_model* m, const float* imgs_dev, float* logits_dev, int32_t F, int32_t H, int32_t W, int32_t group,
                       int32_t flags, void* stream);

/* imgs_dev [F,3,H,W] -> hmaps_dev [F,jnd_out_ch,H,W] */
int vsb_jnd_heatmaps(vsb_model* m, const float* imgs_dev, float* hmaps_dev, int32_t F, int32_t H, int32_t W, void* stream);

/* Host-buffer variants (pinned or pageable): copy in, run, copy out, synchronise. */
int vsb_embed_host(vsb_model* m, const float* imgs_host, const uint8_t* msgs_host, int32_t n_msgs, float* imgs_w_host,
                   float* preds_w_host, int32_t F, int32_t H, int32_t W, int32_t step, int32_t video_mode,
                   int32_t chunk_keys, float scaling_i, float scaling_w, int32_t flags);
int vsb_detect_host(vsb_model* m, const float* imgs_host, float* logits_host, int32_t F, int32_t H, int32_t W, int32_t flags);

/* Streaming form of embed followed by detect of the watermarked frames, HOST (ideally pinned) buffers in and out: the frames are
 * processed in chunks of ~32 with the H2D copy of chunk k+1 and the D2H copy of chunk k-1 overlapped with the compute of chunk k
 * (three internal streams).  This is how the reference's callers use the path on full-resolution video kept on the CPU
 * (evals/full.py:117-120, inference_streaming.py:83-107).  imgs_w_host [F,3,H,W], logits_host [F,1+nbits]. */
int vsb_embed_detect_host(vsb_model* m, const float* imgs_host, const uint8_t* msgs_host, int32_t n_msgs, float* imgs_w_host,
                          float* logits_host, int32_t F, int32_t H, int32_t W, int32_t step, int32_t video_mode,
                          int32_t chunk_keys, float scaling_i, float scaling_w, int32_t flags);

/* The streaming caller's form (inference_streaming.py:23-33 embed_video_clip, :116-124 detect_video_clip): RGB24 frames
 * [F,H,W,3] uint8 on the host, converted on the GPU (x = u8 / 255; u8 = (uint8) trunc(imgs_w * 255)) so that PCIe carries one byte
 * per sample instead of four; same chunked three-stream overlap as vsb_embed_detect_host.
 *   frames_w_host != NULL, logits_host == NULL : embed only            (embed_video_clip)
 *   frames_w_host == NULL, logits_host != NULL : detect the input      (detect_video_clip; msgs_host may be NULL)
 *   both != NULL                               : embed, then detect the re-quantised watermarked frames */
int vsb_frames_host_u8(vsb_model* m, const uint8_t* frames_host, const uint8_t* msgs_host, int32_t n_msgs, uint8_t* frames_w_host,
                       float* logits_host, int32_t F, int32_t H, int32_t W, int32_t step, int32_t video_mode, int32_t chunk_keys,
                       float scaling_i, float scaling_w, int32_t flags);

/* number of kernels launched by this library since the last call with reset != 0 (bench.py's gpu_launches) */
int64_t vsb_launch_count(int32_t reset);

/* per-step CUDA-event profile used by bench.py's roofline leg: enable(1), run steps, read "name\ttotal_ms\tcount\n" lines */
int vsb_profile_enable(int32_t on);
int64_t vsb_profile_read(char* buf, int64_t capacity);

/* ---- image quality (handle-less: no model needed)  <-  evals/metrics.py:38-54 ssim / msssim, i.e. pytorch_msssim.ssim / ms_ssim
 * with size_average=False and the package defaults (11-tap Gaussian window, sigma 1.5, K = (0.01, 0.03), MS-SSIM weights
 * 0.0448 0.2856 0.3001 0.2363 0.1333, avg_pool2d(2, padding = size % 2) between levels, no ReLU on SSIM).
 * x_dev, y_dev [B,C,H,W] fp32 contiguous on one device; ssim_out_dev / msssim_out_dev [B] fp32 on that device, either may be NULL
 * but not both.  An axis shorter than 11 is not filtered (SSIM only); MS-SSIM needs min(H, W) > 160.  The caller supplies a
 * workspace of at least vsb_quality_workspace_bytes(B, C, H, W, msssim_out != NULL) bytes (16-byte aligned; block sums and the
 * pooled levels); nothing is allocated per call.  Deterministic: a frame's values do not depend on B or on the run.  Runs on the
 * pointers' device (the caller's current device is restored); VSB_ERR_UNSUPPORTED on anything but compute capability 9.0.
 * Arguments are checked before any CUDA call, the device match after. */
int64_t vsb_quality_workspace_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t multiscale);   /* host-only; < 0 on error */
int vsb_ssim(const float* x_dev, const float* y_dev, int32_t B, int32_t C, int32_t H, int32_t W, float data_range,
             float* ssim_out_dev, float* msssim_out_dev, void* workspace_dev, int64_t workspace_bytes, void* stream);

/* ---- validation augmentations (handle-less)  <-  augmentation/geometric.py, valuemetric.py as get_validation_augs lists them
 * (evals/full.py:188-239), and video.py's WindowAveraging.  x_dev [B,3,H,W] fp32 contiguous, y_dev [B,3,OH,OW] (OH, OW = H, W for every op but crop, resize
 * and the grid ops); y_dev must not overlap x_dev.  params are host floats, n_params of them:
 *   VSB_AUG_CROP_FLIP      {i, j, flip}: y = x[..., i:i+OH, j:j+OW], mirrored along W when flip != 0      (F.crop, F.hflip)
 *   VSB_AUG_GRID_*         {t00, t01, t10, t11, t20, t21, c6, c7, perspective}: torchvision's rescaled theta [3][2] (and the
 *                          perspective denominator's coefficients); aux_dev holds the base grid, [OW] x then [OH] y values as
 *                          torch.linspace makes them.  grid_sample, align_corners=False, zero padding    (F.rotate, F.perspective)
 *   VSB_AUG_BRIGHTNESS / CONTRAST / SATURATION  {f, 1 - f} rounded to fp32: clamp(f x + (1 - f) o, 0, 1), o = 0, the image's mean
 *                          grayscale, the pixel's grayscale                        (F.adjust_brightness / contrast / saturation)
 *   VSB_AUG_HUE            {hue_factor}                                             (F.adjust_hue)
 *   VSB_AUG_GRAYSCALE      {}: 0.299 r + 0.587 g + 0.114 b on all three channels    (the reference's Grayscale)
 *   VSB_AUG_BLUR           k fp32 taps (k odd, <= 33): the separable form of F.gaussian_blur, reflect padding
 *   VSB_AUG_JPEG           {quality}: PIL's JPEG save and load (4:2:0, islow DCT, fancy upsampling), bit-exact, then the
 *                          reference's pass-through (jpeg - x) + x on the clamped input                    (utils/image.py:13-34)
 *   VSB_AUG_RESIZE         {}: bilinear, antialias=True, align_corners=False, H x W -> OH x OW           (F.resize)
 *   VSB_AUG_WINDOW_AVG     {window, alpha, 1 - alpha}, the two blend factors rounded to fp32 from the caller's doubles: x is a
 *                          clip of B = T frames; with w = min(window, T) and h = w / 2, frame i becomes
 *                          (1 - alpha) x[i] + alpha mean(x[max(0, i - h) : min(T, i + h + 1)]), the mean a fresh fp32 sum in
 *                          frame order over the count (video.py:455-485; an even window spans w + 1 frames inside the clip).
 *                          window is an integer >= 1 and alpha finite (VSB_ERR_INVALID); w > 17 is VSB_ERR_UNSUPPORTED.
 *                          The caller returns a clip of T <= min_window_size unchanged, as the reference's class does.
 *                          x_dev and y_dev need only fp32 (4-byte) alignment: the 16-byte vector path is taken when both are
 *                          16-byte aligned and 3 H W is a multiple of 4, the one-float path otherwise.
 * The caller supplies vsb_augment_workspace_bytes(op, B, H, W) bytes of device workspace (16-byte aligned; 0 = none needed).
 * Deterministic: the contrast mean is a fixed-order fp64 sum.  Runs on x_dev's device; VSB_ERR_UNSUPPORTED on anything but
 * compute capability 9.0; arguments are checked before any CUDA call. */
enum vsb_aug_op {
  VSB_AUG_CROP_FLIP = 0, VSB_AUG_GRID_NEAREST = 1, VSB_AUG_GRID_BILINEAR = 2, VSB_AUG_BRIGHTNESS = 3, VSB_AUG_CONTRAST = 4,
  VSB_AUG_SATURATION = 5, VSB_AUG_HUE = 6, VSB_AUG_GRAYSCALE = 7, VSB_AUG_BLUR = 8, VSB_AUG_JPEG = 9, VSB_AUG_RESIZE = 10,
  VSB_AUG_WINDOW_AVG = 11
};
int64_t vsb_augment_workspace_bytes(int32_t op, int32_t B, int32_t H, int32_t W);   /* host-only; < 0 on error */
int vsb_augment(int32_t op, const float* x_dev, float* y_dev, int32_t B, int32_t C, int32_t H, int32_t W, int32_t OH, int32_t OW,
                const float* params, int32_t n_params, const float* aux_dev, void* workspace_dev, int64_t workspace_bytes, void* stream);

/* ---- debug / test seams (used by tests/ only) ------------------------------------------------------------- */
/* copy a named intermediate activation of the most recent embed/detect sub-batch to the host as fp32.
 * shape4 receives [B, H, W, C] (NHWC) or [M, C, 1, 1]-style dims; returns the element count or <0. */
int64_t vsb_debug_get_tensor(vsb_model* m, const char* name, float* host_out, int64_t capacity, int64_t* shape4);
/* ConvNeXt detect plans: on != 0 adds device-to-device copies of the fp32 residual stream where the blocks read it, so that each
 * kernel can be checked on its own inputs.  The stream is updated in place by every block's pwconv2, so without them the input
 * of a block is kept nowhere.  Taps while on (s = 0..3):
 *   s{s}_ds   the stream right after the stem (s = 0) or the down conv of stage s
 *   s{s}_in   the stream right before the stage's last block (the same copy as s{s}_ds at depth 1)
 * The copies only read the stream: the logits are bit-identical with the seam on and off.  Setting it drops the cached detect
 * plans; off (the default), the plans are built exactly as without the seam.  Taps in every ConvNeXt detect plan:
 *   s{s}_ln (s >= 1) the fp16 LayerNorm'd rows the down conv reads;  s{s}_a / s{s}_g  the last block's dwconv + LN output and
 *   its pwconv1 + GELU output (after the in-place GRN on stages that apply it);  s{s}_w2s  [B, C, 1, 4C] the per-sample GRN-scaled
 *   W2 of stages that fold GRN into the weights;  stage{s}  the stream after stage s;  stage3_16  its fp16 copy the head conv
 *   reads;  head_conv;  head_pooled  [B, 1, 1, C] the LayerNorm + GELU + mean the linear head reads.
 * SAM-ViT detect plans reuse one residual stream, one LayerNorm buffer and one neck buffer; with L the last block, the taps while
 * on are
 *   vit.blk{L}.in    fp32 the stream the last block reads        vit.blk{L}.ln1  fp16 its LayerNorm 1 output (LN2 overwrites it)
 *   vit.blk{L}.mid   fp32 the stream after its attention proj (lin2 updates it in place)
 *   vit.neck1x1      fp32 the neck's 1x1 output (the 3x3 writes into the same buffer)
 * and in every SAM-ViT detect plan: vit.patches [B, G, G, 768] fp16 im2col rows (K order c, r, s);  vit.embed  the stream after
 * the patch GEMM + position table;  vit.blk{L}.qkv / .attn / .ln2 / .hid  the last block's qkv rows, attention output, LayerNorm 2
 * output and GELU hidden rows (fp16);  vit.blk{L}  the stream after it;  vit.x16  its fp16 copy the neck reads;  vit.neck_ln1  the
 * fp16 LayerNorm of the 1x1 output;  vit.neck3x3  fp32 the 3x3 output;  vit.neck  the fp16 map the head reads.
 * HiDDeN plans (embed and detect; setting the seam also drops the cached HiDDeN embed plans) reuse two map buffers and one pre-norm
 * map; while on, copies of the first two layers' outputs and (GroupNorm) pre-norm maps are taps henc.{0,1} / henc.{0,1}.pre and
 * hdec.{0,1} / hdec.{0,1}.pre.  Always: the GroupNorm partials <henc|hdec>.{i}.stats (fp64 pairs as four fp32 words), the last
 * maps henc.{L-1}, hdec.{L-3..L-2}, henc.cat_x (image columns + message table), henc.cat.pre, hdec.{L-1}.pre, henc.msg_table,
 * head_pooled and delta. */
int vsb_debug_keep_inputs(vsb_model* m, int32_t on);
/* host-only: the variant finalize_op chose for each tensor-core step of the most recent plan, one line per step in plan order:
 * "name\tM=..\tN=..\tK=..\tblock_n=..\ttma_store=0|1|2\tb_resident=0|1\tb_fixed_ntile=0|1\tkernel=128|longk\tbias_global=0|1\t
 * m_tiles=whole|ragged\n".  Written like vsb_profile_read: returns the bytes needed (with the terminating 0), or < 0; buf is
 * filled when capacity is at least that. */
int64_t vsb_debug_plan_gemms(vsb_model* m, char* buf, int64_t capacity);
/* which compiled variant the most recent launch of each full-resolution kernel used (host state, no synchronisation):
 *   out[0..4]  resize_sep_kernel:  MT (x taps in registers: 2, 8, or 0 = any count), GST (input rows per staging round: 4, 2, 1),
 *              vec (1 = bulk copies, 0 = 4-byte cp.async), toy (output rows per block), OW (output width = img_size)
 *   out[5..9]  blend:  3 = jnd_blend3_kernel (TMA-fed) or 2 = jnd_blend2_kernel, VEC (4 or 1), FASTUP (1 = delta read in place or
 *              through <= 2 taps per axis, 4 = through 3 or 4 taps per axis (bicubic), 0 = generic tables), CD (delta channels),
 *              JIN (heat-map inputs: 1 luminance, 3 per RGB channel)
 * Entries are -1 until that kernel has run on this handle.  capacity >= 10; returns 10, or < 0. */
int32_t vsb_debug_last_dispatch(vsb_model* m, int32_t* out, int32_t capacity);
/* standalone conv/GEMM on the wgmma kernels for unit tests: see tests/test_conv_gemm_gpu.py */
typedef struct vsb_conv_test {
  int32_t loader;            /* 0 TMA per tap, 1 gather conv, 4 halo conv3x3, 5 direct 3x3 ring conv */
  int32_t B, IH, IW, C0, C1; /* input NHWC fp16 [B,IH,IW,C0] (+ optional second source [.., C1]) */
  int32_t R, S, stride, pad, pad_mode;
  int32_t N;                 /* C_out; weights fp16 [N][R*S*(C0+C1)] */
  int32_t epi, act;          /* 0 affine / 1 LN;  0 none 1 relu 2 gelu */
  int32_t rows_per_sample;   /* GRN */
  int32_t block_n;           /* 0 = auto */
  const void* src0; const void* src1; const void* weights;
  const float* bias; const void* resid16; const float* resid32;
  const float* ln_w; const float* ln_b;
  const float* outc_w; const float* outc_b; int32_t n_out;
  void* out16; float* out32; float* delta; float* grn_stats;
  int32_t ld0;               /* pixel pitch of src0 in elements (0 = C0): widths that are not multiples of 8 live in padded rows */
  int32_t ldw;               /* row pitch of the weights (0 = K) */
  int32_t ld_out;            /* row pitch of out16 / out32 / resid32 (0 = N) */
  int32_t kernel;            /* tensor-core loaders: 0 = the kernel the library selects, 1 = force the 128-row kernel, 2 = force the
                              * 256-row long-K kernel (an error unless the op is one it can run) */
  int32_t* kernel_ran;       /* if not null (host memory): receives 1 or 2, the kernel this call launched */
  int32_t grn_part;          /* with grn_stats: 1 = per-32-row partial rows [M / 32][N] (stored, no atomics), 0 = [samples][N] (atomics) */
  int32_t w_samples;         /* > 1: weights are [w_samples][N][K], sample = GEMM row / rows_per_sample (0 or 1: one weight matrix) */
  int32_t longk_block_n;     /* the 256-row long-K kernel's tile width: 0 = the one the library selects, 128 or 192 = that one (an
                              * error with kernel = 2 unless the op can run at it); block_n sets the 128-row kernel's */
} vsb_conv_test;
int vsb_debug_conv(const vsb_conv_test* t, void* stream);
/* host-only (no GPU needed): the separable table the resize kernels use along one axis of length `in` -> `out`, i.e. the library's
 * restatement of ATen's bilinear (anti-aliased or plain, align_corners=False) index/weight computation behind F.interpolate
 * (wam.py:163,184,224).  start / cnt: [out]; weights: [out * maxt] row-major, capacity in floats.  Returns maxt, or < 0. */
int vsb_debug_resample_table(int32_t in, int32_t out, int32_t antialias, int32_t* start, int32_t* cnt, float* weights, int64_t capacity);
/* the same for any resize the flags describe: mode a vsb_resize_mode, align_corners and antialias 0 / 1 (VSB_ERR_INVALID for the
 * combinations F.interpolate rejects).  Every table has contiguous taps inside [0, in): bicubic taps past an edge are folded into
 * the edge tap's weight.  With mode 0 and align_corners 0 it returns what vsb_debug_resample_table returns. */
int vsb_debug_resample_table2(int32_t in, int32_t out, int32_t mode, int32_t align_corners, int32_t antialias, int32_t* start, int32_t* cnt,
                              float* weights, int64_t capacity);

#ifdef __cplusplus
}
#endif
#endif /* VSB200_H */

/* vf_b200_model.h — MODEL-LEVEL C-ABI of viewformer_b200 (libvf_b200_model.so).
 *
 * The entry points SURVEY.md §8(b) lists for a non-Python host: create a codebook / transformer from a checkpoint directory (or from the
 * reference's initialisers), encode / decode, transformer forward, context prefill + queries, generate().  Plain pointers, sizes and a
 * cudaStream_t; every pointer is a DEVICE pointer unless stated; integer status (0 ok, < 0 error, vf_model_last_error()).
 *
 * Implementation note.  The layer sequencing of the two models is host logic that exists once, in the reference's own language
 * (viewformer_b200/vqgan.py, migt.py).  This library does not restate it: it embeds the CPython interpreter (or re-uses the running one when
 * loaded into a Python process), imports viewformer_b200.cabi and forwards every call with the raw pointers wrapped zero-copy
 * (__cuda_array_interface__) on the caller's stream.  All arithmetic runs in the kernels of libvf_b200.so (vf_b200.h).  A host therefore
 * needs this image's Python environment at run time (VF_PYTHON_EXECUTABLE, default: the interpreter the library was built with) but no
 * Python code of its own.  Calls are serialised by the interpreter lock; one host thread at a time per process is the intended use
 * (the reference's callers are single-threaded Python).  All device work of a call is enqueued on `stream`; outputs are complete when
 * the stream has drained (cudaStreamSynchronize / an event), exactly as with the kernels of vf_b200.h.
 *
 * Reference interfaces replaced:
 *   vf_vq_create            viewformer/utils/torch.py:9-17 (load_model), models/__init__.py:38-59 (AutoModelTH.from_config)
 *   vf_vq_encode            models/vqgan_th.py:379-383 (VQGAN.encode()[-1]); uint8 NHWC entry: evaluate/evaluate_transformer.py:105-110
 *   vf_vq_decode_code       models/vqgan_th.py:390-393; uint8 NHWC exit: evaluate_transformer.py:127-129
 *   vf_migt_create          viewformer/utils/tensorflow.py:20-63 (load_model), models/__init__.py:15-35
 *   vf_migt_forward         models/migt.py:338-455 (MIGT.call, single stream, training=False), evaluate_transformer.py:118-123
 *   vf_migt_prefill_context / vf_migt_query   evaluate/evaluate_transformer_multictx_allimg.py:141-173 (one context, many queries)
 *   vf_generate             evaluate/evaluate_transformer.py:97-146 (generate_batch_predictions)
 */
#ifndef VF_B200_MODEL_H
#define VF_B200_MODEL_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef int64_t vf_handle_t;          /* > 0; 0 is never a valid handle */
typedef void* vf_cuda_stream_t;       /* cudaStream_t; NULL = the device's current torch stream */

enum { VF_LAYOUT_U8_NHWC = 0, VF_LAYOUT_F32_NCHW = 1, VF_LAYOUT_F32_NHWC = 2 };

/* Starts (or attaches to) the interpreter and imports viewformer_b200.  Called implicitly by every other entry point. */
int vf_model_init(void);
const char* vf_model_last_error(void);

/* checkpoint_dir: directory with config.json + weights (Lightning .ckpt for the codebook, TF2 object-graph checkpoint or .ckpt for the
 * transformer).  NULL / "": reference initialisers under `seed`, configuration = config_json (models/config.py keys; NULL = defaults).
 * precision: "mixed" (codebook default: bit-exact codes, bf16 decoder), "bf16", "tf32", "fp32".  device: CUDA ordinal. */
int vf_vq_create(const char* config_json, const char* checkpoint_dir, const char* precision, int device, int64_t seed, vf_handle_t* out);
int vf_vq_info(vf_handle_t h, int* image_size, int* tokens_per_side, int* n_embed, int* in_channels);
/* images: [n,S,S,C] uint8 / [n,C,S,S] f32 in [-1,1] / [n,S,S,C] f32 per `layout`; codes: int64 [n,s,s].  C is the codebook's
 * in_channels (vf_vq_info: 3 for RGB, 4 for RGB + mask) for vf_vq_encode, its out_ch (equal in every released codebook) for
 * vf_vq_decode_code. */
int vf_vq_encode(vf_handle_t h, const void* images, int layout, int n, int64_t* codes, vf_cuda_stream_t stream);
int vf_vq_decode_code(vf_handle_t h, const int64_t* codes, int n, void* images, int layout, vf_cuda_stream_t stream);

int vf_migt_create(const char* config_json, const char* checkpoint_dir, const char* precision, int device, int64_t seed, vf_handle_t* out);
int vf_migt_info(vf_handle_t h, int* tokens_per_side, int* n_embeddings, int* mask_token, int* use_localization);
/* input_ids int32 [B,T,s,s] (mask_token in the views to generate), poses f32 [B,T,7] (relative, normalised).
 * codes_last int64 [B,s,s] = argmax of the last view; logits_last f32 [B,s,s,n_embeddings] or NULL. */
int vf_migt_forward(vf_handle_t h, const int32_t* input_ids, const float* poses, int B, int T, int64_t* codes_last, float* logits_last,
                    vf_cuda_stream_t stream);
/* KV cache over Tc context views (BASELINE configs[4]); the cache handle is released with vf_destroy */
int vf_migt_prefill_context(vf_handle_t h, const int32_t* context_ids, const float* context_poses, int B, int Tc, vf_handle_t* cache,
                            vf_cuda_stream_t stream);
/* query_poses f32 [Nq,7]; Nq = B of the cache (one query per scene) or any Nq when the cache holds one scene; codes int64 [Nq,s,s] */
int vf_migt_query(vf_handle_t h, vf_handle_t cache, const float* query_poses, int Nq, int64_t* codes, vf_cuda_stream_t stream);

/* images uint8 [B,T,S,S,in_channels], cameras f32 [B,T,7] (world poses: xyz + wxyz quaternion) -> generated_images uint8 [B,S,S,out_ch],
 * generated_cameras f32 [B,7] (NULL to skip; written only by localising models) */
int vf_generate(vf_handle_t transformer, vf_handle_t codebook, const uint8_t* images, const float* cameras, int B, int T,
                uint8_t* generated_images, float* generated_cameras, vf_cuda_stream_t stream);

int vf_destroy(vf_handle_t h);

#ifdef __cplusplus
}
#endif
#endif

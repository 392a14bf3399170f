/*
 * minigpt4.h — C ABI of the H100-native MiniGPT-4 engine (libminigpt4.so).
 *
 * This header re-declares, symbol for symbol and field for field, the drop-in
 * boundary of Maknee/minigpt4.cpp so that the unmodified ctypes binding
 * (reference minigpt4/minigpt4_library.py:94-227) and the example CLI
 * (reference examples/main.cpp:207-293) bind to the new library.
 * Every declaration cites the reference interface it replaces (minigpt4.h:LINE).
 * Enumerator ORDER is ABI: callers pass plain ints.
 */
#ifndef MINIGPT4_B200_ABI_H
#define MINIGPT4_B200_ABI_H

#include <stddef.h>
#include <stdint.h>
#include <stdbool.h>

#if defined(_WIN32)
#  define MINIGPT4_API __declspec(dllexport)
#else
#  define MINIGPT4_API __attribute__((visibility("default")))
#endif

#ifndef IN
#  define IN
#endif
#ifndef OUT
#  define OUT
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* opaque engine handle (reference minigpt4.h:28) */
struct MiniGPT4Context;

/* tensor dtype ids used in the model container and by minigpt4_quantize_model
 * (reference minigpt4.h:30-48; NOT ggml's numbering) */
enum MiniGPT4DataType {
    F16 = 0, F32 = 1, I32 = 2, L64 = 3,
    Q4_0 = 4, Q4_1 = 5, Q5_0 = 6, Q5_1 = 7, Q8_0 = 8, Q8_1 = 9,
    Q2_K = 10, Q3_K = 11, Q4_K = 12, Q5_K = 13, Q6_K = 14, Q8_K = 15
};

/* reference minigpt4.h:50-56 */
enum MiniGPT4Verbosity {
    MINIGPT4_VERBOSITY_NONE = 0,
    MINIGPT4_VERBOSITY_ERROR = 1,
    MINIGPT4_VERBOSITY_INFO = 2,
    MINIGPT4_VERBOSITY_DEBUG = 3
};

/* reference minigpt4.h:58-63 */
enum MiniGPT4ImageFormat {
    MINIGPT4_IMAGE_FORMAT_UNKNOWN = 0,
    MINIGPT4_IMAGE_FORMAT_F32 = 1,
    MINIGPT4_IMAGE_FORMAT_U8 = 2
};

/* reference minigpt4.h:65-72 — caller-owned pixel buffer; for encode it must be
 * F32, planar CHW, 3x224x224 */
struct MiniGPT4Image {
    void *data;
    int width;
    int height;
    int channels;
    enum MiniGPT4ImageFormat format;
};

/* reference minigpt4.h:74-78 — host float buffer, 32 rows x n_embd_llm */
struct MiniGPT4Embedding {
    float *data;
    size_t elements;
};

/* reference minigpt4.h:80-90 — plural carriers (unused by the reference's 18
 * entry points; used by the batch extension in minigpt4_b200.h) */
struct MiniGPT4Embeddings {
    struct MiniGPT4Embedding *embeddings;
    size_t n_embeddings;
};
struct MiniGPT4Images {
    struct MiniGPT4Image *images;
    size_t n_images;
};

/* reference minigpt4.h:92-95 */
enum MiniGPT4ImageLoadFlags { MINIGPT4_IMAGE_LOAD_FLAG_NONE = 0 };

/* --- the 18 entry points (reference minigpt4.h:97-114) --------------------- */

/* minigpt4.h:97 — load MiniGPT-4 container + ggjt LLaMA file into HBM; NULL on failure */
MINIGPT4_API struct MiniGPT4Context *minigpt4_model_load(const char *path, const char *llm_model,
                                                         int verbosity, int seed, int n_ctx,
                                                         int n_batch, bool numa);
/* minigpt4.h:98-99 — OpenCV-only in the reference (minigpt4.cpp:2576-2651; its default build returns OpenCVNotLinked).
 * Here: PNG / JPEG / PPM / PGM file -> 8-bit RGB (OpenImage (5) for anything else), then Pillow-bicubic resize to 224x224,
 * /255, CLIP mean/std, planar CHW F32 - the tensor minigpt4_encode_image takes. Release both with minigpt4_free_image. */
MINIGPT4_API int minigpt4_image_load_from_file(struct MiniGPT4Context *ctx, const char *path,
                                               IN struct MiniGPT4Image *image, int flags);
MINIGPT4_API int minigpt4_preprocess_image(struct MiniGPT4Context *ctx,
                                           IN const struct MiniGPT4Image *image,
                                           OUT struct MiniGPT4Image *preprocessed_image, int flags);
/* minigpt4.h:100 — ViT-g/14 + Q-Former + llama_proj forward */
MINIGPT4_API int minigpt4_encode_image(struct MiniGPT4Context *ctx, IN struct MiniGPT4Image *image,
                                       OUT struct MiniGPT4Embedding *embedding, size_t n_threads);
/* minigpt4.h:101 — "Human: <Img>" + 32 embedding rows + "</Img> " + s + "### Assistant:" */
MINIGPT4_API int minigpt4_begin_chat_image(struct MiniGPT4Context *ctx,
                                           IN struct MiniGPT4Embedding *image_embedding,
                                           const char *s, size_t n_threads);
/* minigpt4.h:102 — sample one token, return its text, feed it back (one decode step) */
MINIGPT4_API int minigpt4_end_chat_image(struct MiniGPT4Context *ctx, const char **token,
                                         size_t n_threads, float temp, int32_t top_k, float top_p,
                                         float tfs_z, float typical_p, int32_t repeat_last_n,
                                         float repeat_penalty, float alpha_presence,
                                         float alpha_frequency, int mirostat, float mirostat_tau,
                                         float mirostat_eta, int penalize_nl);
/* minigpt4.h:103 */
MINIGPT4_API int minigpt4_system_prompt(struct MiniGPT4Context *ctx, size_t n_threads);
/* minigpt4.h:104 — "Human: " + s + "### Assistant:" */
MINIGPT4_API int minigpt4_begin_chat(struct MiniGPT4Context *ctx, const char *s, size_t n_threads);
/* minigpt4.h:105 — alias of end_chat_image */
MINIGPT4_API int minigpt4_end_chat(struct MiniGPT4Context *ctx, const char **token, size_t n_threads,
                                   float temp, int32_t top_k, float top_p, float tfs_z,
                                   float typical_p, int32_t repeat_last_n, float repeat_penalty,
                                   float alpha_presence, float alpha_frequency, int mirostat,
                                   float mirostat_tau, float mirostat_eta, int penalize_nl);
/* minigpt4.h:106 — n_past = 0 */
MINIGPT4_API int minigpt4_reset_chat(struct MiniGPT4Context *ctx);
/* minigpt4.h:107-108 — return EosToken(11)/Eos(12) as "true", 0 otherwise */
MINIGPT4_API int minigpt4_contains_eos_token(const char *s);
MINIGPT4_API int minigpt4_is_eos(const char *s);
/* minigpt4.h:109-111 */
MINIGPT4_API int minigpt4_free(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_free_image(struct MiniGPT4Image *image);
MINIGPT4_API int minigpt4_free_embedding(struct MiniGPT4Embedding *embedding);
/* minigpt4.h:112 — enumerator name of MiniGPT4Error */
MINIGPT4_API const char *minigpt4_error_code_to_string(int error_code);
/* minigpt4.h:113 — container -> container quantiser */
MINIGPT4_API int minigpt4_quantize_model(const char *in_path, const char *out_path, int data_type);
/* minigpt4.h:114 */
MINIGPT4_API void minigpt4_set_verbosity(int verbosity);

#ifdef __cplusplus
}
#endif
#endif /* MINIGPT4_B200_ABI_H */

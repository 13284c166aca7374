/* lfd_detect -- runs a model file on raw video frames with liblfd_b200.so and cudart alone (no Python, no torch).
 *
 *     lfd_detect MODEL FRAMES HEIGHT WIDTH [bgr|gray|nv12] [--scale S]
 *
 * MODEL   a model file written by lfd.deployment.export_model (include/lfd_b200.h, "model files")
 * FRAMES  raw uint8 frames of HEIGHT x WIDTH back to back: the model's own kind by default -- BGR (HEIGHT * WIDTH * 3 bytes each) for a
 *         model whose image op (op 0) has Cin = 3, gray (HEIGHT * WIDTH bytes each) for one with Cin = 1 -- or NV12 (a Y plane of
 *         HEIGHT x WIDTH bytes, then the interleaved UV plane of HEIGHT / 2 x WIDTH bytes; a gray model reads the Y plane only);
 *         HEIGHT and WIDTH at most the model's capacity
 * --scale S  the frames are of any size and are resized on the GPU by S (lfd_engine_detect_resized), as cv2.resize(frame, (0, 0), fx=S,
 *         fy=S) would resize them; the resized size must fit the model's capacity.  The rows are in the frames' own coordinates, those
 *         of the reference's get_results with meta resize_scale S, resized_height int(HEIGHT * S), resized_width int(WIDTH * S).
 *
 * The frames run in batches of the model's N (a last partial batch is padded with black frames, whose rows are not printed).  For every
 * frame it prints "frame INDEX COUNT" and then COUNT rows "label score x y w h" -- the rows of LFD.predict_for_single_image, with
 * w = x2 - x1 + 1 and h = y2 - y1 + 1 in float32 -- every float with %.9g, which reads back to the same float. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "lfd_b200.h"

#define CHECK_LFD(call)                                                                        \
    do {                                                                                       \
        int rc_ = (call);                                                                      \
        if (rc_ != LFD_OK) {                                                                   \
            fprintf(stderr, "%s failed (%d): %s\n", #call, rc_, lfd_last_error());            \
            return 1;                                                                          \
        }                                                                                      \
    } while (0)
#define CHECK_CUDA(call)                                                                       \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) {                                                               \
            fprintf(stderr, "%s failed: %s\n", #call, cudaGetErrorString(e_));                \
            return 1;                                                                          \
        }                                                                                      \
    } while (0)

static void* read_file(const char* path, size_t* n) {
    FILE* f = fopen(path, "rb");
    if (!f) return NULL;
    fseek(f, 0, SEEK_END);
    long size = ftell(f);
    fseek(f, 0, SEEK_SET);
    void* buf = malloc(size > 0 ? (size_t)size : 1);
    if (buf && size > 0 && fread(buf, 1, (size_t)size, f) != (size_t)size) {
        free(buf);
        buf = NULL;
    }
    fclose(f);
    *n = size > 0 ? (size_t)size : 0;
    return buf;
}

int main(int argc, char** argv) {
    double scale = 0.0;   /* 0: the frames run at their own size */
    if (argc >= 7 && strcmp(argv[argc - 2], "--scale") == 0) {
        char* end = NULL;
        scale = strtod(argv[argc - 1], &end);
        if (!end || *end || !(scale > 0.0)) {
            fprintf(stderr, "--scale takes a number > 0, got %s\n", argv[argc - 1]);
            return 2;
        }
        argc -= 2;
    }
    if (argc < 5 || argc > 6) {
        fprintf(stderr, "usage: %s MODEL FRAMES HEIGHT WIDTH [bgr|gray|nv12] [--scale S]\n", argv[0]);
        return 2;
    }
    const int h = atoi(argv[3]), w = atoi(argv[4]);
    const int nv12 = argc == 6 && strcmp(argv[5], "nv12") == 0;
    if (argc == 6 && !nv12 && strcmp(argv[5], "bgr") != 0 && strcmp(argv[5], "gray") != 0) {
        fprintf(stderr, "frame format must be bgr, gray or nv12, got %s\n", argv[5]);
        return 2;
    }
    size_t model_bytes = 0, frames_bytes = 0;
    void* model = read_file(argv[1], &model_bytes);
    uint8_t* frames = (uint8_t*)read_file(argv[2], &frames_bytes);
    if (!model || !frames) {
        fprintf(stderr, "cannot read %s\n", model ? argv[2] : argv[1]);
        return 1;
    }
    lfd_engine* engine = NULL;
    CHECK_LFD(lfd_engine_open(model, model_bytes, &engine));
    free(model);
    lfd_engine_desc d;
    CHECK_LFD(lfd_engine_info(engine, &d));
    lfd_op image_op;   /* op 0 reads the frames: Cin = 3 (BGR) or 1 (gray) bytes per pixel of a uint8 frame */
    int32_t src_op, level;
    CHECK_LFD(lfd_engine_op(engine, 0, &image_op, &src_op, &level));
    const size_t px = (size_t)image_op.Cin;
    if (argc == 6 && !nv12 && (strcmp(argv[5], "gray") == 0) != (px == 1)) {
        fprintf(stderr, "%s frames on a %s model\n", argv[5], px == 1 ? "gray" : "BGR");
        return 2;
    }
    if (h < 1 || w < 1 || (!scale && (h > d.H || w > d.W)) || (nv12 && ((h | w) & 1))) {
        fprintf(stderr, "frames of %dx%d do not fit the model's capacity %dx%d%s\n", h, w, d.H, d.W, nv12 ? " (NV12: even sizes)" : "");
        return 1;
    }
    if (scale) {   /* the size the frames are resized to must fit (lfd_engine_detect_resized checks it too) */
        int rh, rw, mode;
        CHECK_LFD(lfd_resize_query(h, w, scale, &rh, &rw, &mode));
        if (rh > d.H || rw > d.W) {
            fprintf(stderr, "frames of %dx%d at scale %g are %dx%d, beyond the model's capacity %dx%d\n", h, w, scale, rh, rw, d.H, d.W);
            return 1;
        }
    }
    const size_t frame_bytes = nv12 ? (size_t)h * w * 3 / 2 : (size_t)h * w * px;
    /* one image as the device input holds it: the frame itself when it is resized there, else the frame in the capacity layout */
    const size_t image_bytes = scale ? frame_bytes : nv12 ? (size_t)d.H * d.W * 3 / 2 : (size_t)d.H * d.W * px;
    const size_t n_frames = frames_bytes / frame_bytes;
    if (n_frames * frame_bytes != frames_bytes) {
        fprintf(stderr, "%s holds %zu bytes, not a whole number of %zu-byte frames\n", argv[2], frames_bytes, frame_bytes);
        return 1;
    }

    void *weights, *workspace, *post_workspace, *input, *resized = NULL;
    float* dets;
    int32_t *labels, *count;
    const size_t cap = (size_t)d.cap;
    CHECK_CUDA(cudaMalloc(&weights, (size_t)d.weights_bytes));
    CHECK_CUDA(cudaMalloc(&workspace, (size_t)d.workspace_bytes));
    CHECK_CUDA(cudaMalloc(&post_workspace, (size_t)d.post_workspace_bytes));
    CHECK_CUDA(cudaMalloc(&input, d.N * image_bytes));
    if (scale) CHECK_CUDA(cudaMalloc(&resized, (size_t)d.N * d.H * d.W * px));   /* the resized frames, capacity layout */
    CHECK_CUDA(cudaMalloc((void**)&dets, d.N * cap * 5 * sizeof(float)));
    CHECK_CUDA(cudaMalloc((void**)&labels, d.N * cap * sizeof(int32_t)));
    CHECK_CUDA(cudaMalloc((void**)&count, (d.N + 1) * sizeof(int32_t)));
    cudaStream_t stream;
    CHECK_CUDA(cudaStreamCreate(&stream));
    CHECK_LFD(lfd_engine_bind(engine, weights, (size_t)d.weights_bytes, workspace, (size_t)d.workspace_bytes, post_workspace,
                              (size_t)d.post_workspace_bytes, stream));

    uint8_t* batch = (uint8_t*)calloc(d.N, image_bytes);
    float* host_dets = (float*)malloc(d.N * cap * 5 * sizeof(float));
    int32_t* host_labels = (int32_t*)malloc(d.N * cap * sizeof(int32_t));
    int32_t* host_count = (int32_t*)malloc((d.N + 1) * sizeof(int32_t));
    if (!batch || !host_dets || !host_labels || !host_count) {
        fprintf(stderr, "out of host memory\n");
        return 1;
    }
    for (size_t first = 0; first < n_frames; first += (size_t)d.N) {
        /* the frames of the batch in the top-left corner of the capacity layout (lfd_plan_forward_extent) */
        memset(batch, 0, d.N * image_bytes);
        for (int i = 0; i < d.N && first + i < n_frames; ++i) {
            const uint8_t* f = frames + (first + i) * frame_bytes;
            uint8_t* img = batch + i * image_bytes;
            if (scale) {
                memcpy(img, f, frame_bytes);
            } else if (nv12) {
                for (int r = 0; r < h; ++r) memcpy(img + (size_t)r * d.W, f + (size_t)r * w, (size_t)w);
                for (int r = 0; r < h / 2; ++r) memcpy(img + (size_t)(d.H + r) * d.W, f + (size_t)(h + r) * w, (size_t)w);
            } else {
                for (int r = 0; r < h; ++r) memcpy(img + (size_t)r * d.W * px, f + (size_t)r * w * px, (size_t)w * px);
            }
        }
        CHECK_CUDA(cudaMemcpyAsync(input, batch, d.N * image_bytes, cudaMemcpyHostToDevice, stream));
        if (scale)
            CHECK_LFD(lfd_engine_detect_resized(engine, input, nv12 ? LFD_INPUT_U8_NV12 : LFD_INPUT_U8_NHWC, h, w, scale, (uint8_t*)resized, dets,
                                                labels, count, NULL, NULL, 1, stream));
        else
            CHECK_LFD(lfd_engine_detect(engine, input, nv12 ? LFD_INPUT_U8_NV12 : LFD_INPUT_U8_NHWC, h, w, dets, labels, count, NULL, NULL, 1, stream));
        CHECK_CUDA(cudaMemcpyAsync(host_dets, dets, d.N * cap * 5 * sizeof(float), cudaMemcpyDeviceToHost, stream));
        CHECK_CUDA(cudaMemcpyAsync(host_labels, labels, d.N * cap * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
        CHECK_CUDA(cudaMemcpyAsync(host_count, count, (d.N + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
        CHECK_CUDA(cudaStreamSynchronize(stream));
        if (host_count[d.N]) {
            fprintf(stderr, "more than %d candidates passed the score threshold in one image\n", d.cap);
            return 1;
        }
        for (int i = 0; i < d.N && first + i < n_frames; ++i) {
            printf("frame %zu %d\n", first + i, host_count[i]);
            for (int k = 0; k < host_count[i]; ++k) {
                const float* b = host_dets + ((size_t)i * cap + k) * 5;
                const float bw = (b[2] - b[0]) + 1.0f, bh = (b[3] - b[1]) + 1.0f;
                printf("%d %.9g %.9g %.9g %.9g %.9g\n", host_labels[(size_t)i * cap + k], b[4], b[0], b[1], bw, bh);
            }
        }
    }
    lfd_engine_close(engine);
    cudaStreamDestroy(stream);
    cudaFree(weights);
    cudaFree(workspace);
    cudaFree(post_workspace);
    cudaFree(input);
    cudaFree(resized);
    cudaFree(dets);
    cudaFree(labels);
    cudaFree(count);
    free(batch);
    free(frames);
    free(host_dets);
    free(host_labels);
    free(host_count);
    return 0;
}

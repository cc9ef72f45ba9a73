/*
 * dd3d_infer -- run DD3D on one image from a self-contained model file, through the C ABI alone.
 *
 *   dd3d_infer [-g] MODEL_FILE IMAGE H W fx s cx 0 fy cy 0 0 1
 *
 * MODEL_FILE: written by DD3DB200.save_model_file.  IMAGE: H * W * 3 bytes, uint8 BGR in CHW order (the layout of the
 * Python model's input["image"]).  The nine numbers: the 3x3 intrinsics, row-major.  Prints one line per detection:
 *
 *   cls score score_3d x1 y1 x2 y2 quat_w quat_x quat_y quat_z proj_ctr_x proj_ctr_y depth W L H loc_x loc_y level attr speed
 *
 * with boxes in the pixel coordinates of the image (option "do_postprocess" on, output size = input size).  Floats print
 * with 9 significant digits, enough to read back the exact fp32 value.
 *
 * -g: the per-frame loop of a deployment instead of dd3d_forward_host: device buffers the program owns, one forward
 * recorded as a CUDA graph (dd3d_graph_create), then per frame write the inputs, dd3d_graph_launch, read the detections
 * back.  Same output.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime.h>

#include "dd3d_b200.h"

static int fail(const char* what, int status, dd3d_handle h) {
    fprintf(stderr, "dd3d_infer: %s failed (%d): %s\n", what, status, dd3d_last_error(h));
    dd3d_destroy(h);
    return 1;
}

/* One frame through a captured forward: device buffers, dd3d_graph_create, H2D, dd3d_graph_launch, D2H. */
static int run_graph(dd3d_handle h, const unsigned char* image, size_t image_bytes, const float* K, const int32_t* sizes,
                     dd3d_det* dets, int cap, int32_t* count) {
    void *d_image = NULL, *d_K = NULL, *d_sizes = NULL, *d_dets = NULL, *d_count = NULL;
    dd3d_graph g = NULL;
    int st = DD3D_ERR_CUDA;
    if (cudaMalloc(&d_image, image_bytes) != cudaSuccess || cudaMalloc(&d_K, 9 * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&d_sizes, 4 * sizeof(int32_t)) != cudaSuccess ||
        cudaMalloc(&d_dets, sizeof(dd3d_det) * (size_t)cap) != cudaSuccess ||
        cudaMalloc(&d_count, sizeof(int32_t)) != cudaSuccess) {
        fprintf(stderr, "dd3d_infer: cudaMalloc failed\n");
        goto done;
    }
    if ((st = dd3d_graph_create(h, d_image, DD3D_IMG_U8, d_K, d_sizes, d_dets, d_count, NULL, &g)) != DD3D_OK) {
        fprintf(stderr, "dd3d_infer: dd3d_graph_create failed (%d): %s\n", st, dd3d_last_error(h));
        goto done;
    }
    /* the per-frame loop, here one frame: write the bound input buffers, launch, read back */
    st = DD3D_ERR_CUDA;
    if (cudaMemcpy(d_image, image, image_bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d_K, K, 9 * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d_sizes, sizes, 4 * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) {
        fprintf(stderr, "dd3d_infer: cudaMemcpy failed\n");
        goto done;
    }
    if ((st = dd3d_graph_launch(g, NULL)) != DD3D_OK) {
        fprintf(stderr, "dd3d_infer: dd3d_graph_launch failed (%d): %s\n", st, dd3d_last_error(h));
        goto done;
    }
    st = DD3D_ERR_CUDA;
    if (cudaMemcpy(count, d_count, sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(dets, d_dets, sizeof(dd3d_det) * (size_t)cap, cudaMemcpyDeviceToHost) != cudaSuccess) {
        fprintf(stderr, "dd3d_infer: cudaMemcpy failed\n");
        goto done;
    }
    st = DD3D_OK;
done:
    dd3d_graph_destroy(g);
    cudaFree(d_image);
    cudaFree(d_K);
    cudaFree(d_sizes);
    cudaFree(d_dets);
    cudaFree(d_count);
    return st;
}

int main(int argc, char** argv) {
    const char* prog = argv[0];
    const int graph = argc > 1 && strcmp(argv[1], "-g") == 0;
    argv += graph;
    argc -= graph;
    if (argc != 14) {
        fprintf(stderr, "usage: %s [-g] MODEL_FILE IMAGE H W k00 k01 k02 k10 k11 k12 k20 k21 k22\n", prog);
        return 2;
    }
    const int H = atoi(argv[3]), W = atoi(argv[4]);
    if (H < 1 || W < 1) {
        fprintf(stderr, "dd3d_infer: bad image size %s x %s\n", argv[3], argv[4]);
        return 2;
    }
    float K[9];
    for (int i = 0; i < 9; ++i) K[i] = strtof(argv[5 + i], NULL);

    const size_t image_bytes = (size_t)3 * H * W;
    unsigned char* image = malloc(image_bytes);
    FILE* f = fopen(argv[2], "rb");
    const int image_ok = image && f && fread(image, 1, image_bytes, f) == image_bytes && fgetc(f) == EOF;
    if (f) fclose(f);
    if (!image_ok) {
        fprintf(stderr, "dd3d_infer: %s is not a %d x %d x 3 byte image\n", argv[2], H, W);
        return 2;
    }

    dd3d_handle h = NULL;
    int st = dd3d_create_from_file(argv[1], &h);
    if (st != DD3D_OK) return fail("dd3d_create_from_file", st, NULL);
    if ((st = dd3d_plan(h, 1, H, W, NULL, 0)) != DD3D_OK) return fail("dd3d_plan", st, h);
    if ((st = dd3d_set_option(h, "do_postprocess", 1)) != DD3D_OK) return fail("dd3d_set_option", st, h);

    const int cap = dd3d_out_cap(h);
    if (cap < 1) return fail("dd3d_out_cap", cap, h);
    dd3d_det* dets = malloc(sizeof(dd3d_det) * (size_t)cap);
    const int32_t sizes[4] = {H, W, H, W}; /* valid size, size the boxes are rescaled to */
    int32_t count = 0, flags = 0;
    if (!dets) return fail("malloc", 0, h);
    if (graph) {
        if (run_graph(h, image, image_bytes, K, sizes, dets, cap, &count) != DD3D_OK) {
            dd3d_destroy(h);
            return 1;
        }
    } else {
        st = dd3d_forward_host(h, image, DD3D_IMG_U8, K, sizes, dets, &count, NULL);
        if (st != DD3D_OK) return fail("dd3d_forward_host", st, h);
    }
    if ((st = dd3d_overflow_flags(h, NULL, &flags)) != DD3D_OK) return fail("dd3d_overflow_flags", st, h);
    if (flags != 0) {
        fprintf(stderr, "dd3d_infer: detection capacity exceeded (flags %d)\n", flags);
        dd3d_destroy(h);
        return 1;
    }

    printf("%d detections\n", count);
    for (int i = 0; i < count; ++i) {
        const dd3d_det* d = &dets[i];
        printf("%d %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g %d %d %.9g\n",
               d->cls, d->score, d->score_3d, d->box[0], d->box[1], d->box[2], d->box[3], d->quat[0], d->quat[1],
               d->quat[2], d->quat[3], d->proj_ctr[0], d->proj_ctr[1], d->depth, d->size[0], d->size[1], d->size[2],
               d->loc[0], d->loc[1], d->level, d->attr, d->speed);
    }
    free(dets);
    free(image);
    dd3d_destroy(h);
    return 0;
}

/* Plain-C client of the hand3d_b200 C ABI (include/hand3d_b200.h): no Python, no PyTorch.
 *
 *   gcc -O2 -Iinclude examples/c_abi_smoke.c -o c_abi_smoke -Lhand3d_b200 -lhand3d_b200 -L/usr/local/cuda/lib64 -lcudart -lm \
 *       -Wl,-rpath,$PWD/hand3d_b200
 *
 * Runs bone_rel_trafo_inv, the TF1-legacy bilinear resize, the mask post-processing and a small fp32 convolution with
 * known answers; exits 0 on success.  Without an sm_90a device h3d_create() must fail with H3D_ENODEVICE (exit code 77).
 */
#include <cuda_runtime_api.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "hand3d_b200.h"

#define CHECK(call)                                                                   \
    do {                                                                              \
        int rc_ = (call);                                                             \
        if (rc_ != H3D_OK) { fprintf(stderr, "%s -> %d: %s\n", #call, rc_, h3d_last_error()); return 1; } \
    } while (0)
#define CU(call)                                                                      \
    do {                                                                              \
        cudaError_t e_ = (call);                                                      \
        if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #call, cudaGetErrorString(e_)); return 1; } \
    } while (0)

int main(void) {
    h3d_ctx* ctx = NULL;
    int rc = h3d_create(&ctx, 0);
    if (rc == H3D_ENODEVICE) { printf("no sm_90a device: %s\n", h3d_last_error()); return 77; }
    if (rc != H3D_OK) { fprintf(stderr, "h3d_create: %s\n", h3d_last_error()); return 1; }
    printf("hand3d_b200 C ABI version %d\n", h3d_version());

    /* 1. bone_rel_trafo_inv: every bone length 1, no articulation -> finger tips at z = 4 */
    float rel[63], xyz[63], *d_rel, *d_xyz;
    for (int i = 0; i < 21; ++i) { rel[3 * i] = 1.f; rel[3 * i + 1] = 0.f; rel[3 * i + 2] = 0.f; }
    CU(cudaMalloc((void**)&d_rel, sizeof rel)); CU(cudaMalloc((void**)&d_xyz, sizeof xyz));
    CU(cudaMemcpy(d_rel, rel, sizeof rel, cudaMemcpyHostToDevice));
    CHECK(h3d_bone_rel_trafo_inv(ctx, d_rel, d_xyz, 1, NULL));
    CU(cudaMemcpy(xyz, d_xyz, sizeof xyz, cudaMemcpyDeviceToHost));
    if (fabsf(xyz[3 * 1 + 2] - 4.f) > 1e-5f || fabsf(xyz[3 * 4 + 2] - 1.f) > 1e-5f || fabsf(xyz[2] - 1.f) > 1e-5f) {
        fprintf(stderr, "bone_rel_trafo_inv: unexpected %f %f %f\n", xyz[5], xyz[14], xyz[2]); return 1;
    }

    /* 2. TF1 legacy bilinear resize: [0, 10] -> 4 samples = [0, 5, 10, 10] (SURVEY.md 9.3) */
    float in2[2] = {0.f, 10.f}, out4[4], *d_in, *d_out;
    CU(cudaMalloc((void**)&d_in, sizeof in2)); CU(cudaMalloc((void**)&d_out, sizeof out4));
    CU(cudaMemcpy(d_in, in2, sizeof in2, cudaMemcpyHostToDevice));
    CHECK(h3d_resize_bilinear_tf1(ctx, d_in, d_out, 1, 1, 2, 1, 1, 4, NULL));
    CU(cudaMemcpy(out4, d_out, sizeof out4, cudaMemcpyDeviceToHost));
    if (out4[0] != 0.f || out4[1] != 5.f || out4[2] != 10.f || out4[3] != 10.f) { fprintf(stderr, "resize KAT failed\n"); return 1; }

    /* 3. mask post-processing: a 11 x 41 foreground rectangle -> center (15, 50), size 40, scale 5 (clipped) */
    const int H = 64, W = 96;
    float* logits = (float*)calloc((size_t)H * W * 2, sizeof(float));
    for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x) {
        logits[(y * W + x) * 2] = 1.f;
        logits[(y * W + x) * 2 + 1] = (y >= 10 && y <= 20 && x >= 30 && x <= 70) ? 3.f : -3.f;
    }
    logits[(12 * W + 33) * 2 + 1] = 9.f;   /* the seed */
    float *d_log, *d_center, *d_size, *d_scale, center[2], size, scale;
    int32_t* d_loc; int32_t loc[2];
    CU(cudaMalloc((void**)&d_log, (size_t)H * W * 2 * 4)); CU(cudaMalloc((void**)&d_center, 8)); CU(cudaMalloc((void**)&d_size, 4));
    CU(cudaMalloc((void**)&d_scale, 4)); CU(cudaMalloc((void**)&d_loc, 8));
    CU(cudaMemcpy(d_log, logits, (size_t)H * W * 2 * 4, cudaMemcpyHostToDevice));
    CHECK(h3d_seg_postprocess(ctx, d_log, 1, H, W, NULL, d_loc, d_center, d_size, d_scale, NULL));
    CU(cudaMemcpy(center, d_center, 8, cudaMemcpyDeviceToHost)); CU(cudaMemcpy(&size, d_size, 4, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&scale, d_scale, 4, cudaMemcpyDeviceToHost)); CU(cudaMemcpy(loc, d_loc, 8, cudaMemcpyDeviceToHost));
    if (center[0] != 15.f || center[1] != 50.f || size != 40.f || scale != 5.f || loc[0] != 12 || loc[1] != 33) {
        fprintf(stderr, "seg_postprocess: center (%g, %g) size %g scale %g loc (%d, %d)\n", center[0], center[1], size, scale, loc[0], loc[1]);
        return 1;
    }

    /* 4. NetworkOps.conv with stride 2 'SAME': [a b c d] * (w0 w1 w2) -> [w0 a + w1 b + w2 c, w0 c + w1 d] (SURVEY.md 9.1) */
    float xin[4] = {1.f, 2.f, 3.f, 5.f}, wk[3] = {0.5f, -1.f, 2.f}, bias = 0.f, yout[2], *d_x, *d_w, *d_b, *d_y;
    CU(cudaMalloc((void**)&d_x, 16)); CU(cudaMalloc((void**)&d_w, 12 * 3)); CU(cudaMalloc((void**)&d_b, 4)); CU(cudaMalloc((void**)&d_y, 8));
    float w33[9] = {0, 0, 0, 0.5f, -1.f, 2.f, 0, 0, 0};      /* 3x3 kernel whose middle row carries the 1-D taps; H = 1 */
    (void)wk;
    CU(cudaMemcpy(d_x, xin, 16, cudaMemcpyHostToDevice)); CU(cudaMemcpy(d_w, w33, 36, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d_b, &bias, 4, cudaMemcpyHostToDevice));
    CHECK(h3d_conv2d_f32(ctx, d_x, d_w, d_b, d_y, 1, 1, 4, 1, 1, 3, 2, 0, NULL));
    CU(cudaMemcpy(yout, d_y, 8, cudaMemcpyDeviceToHost));
    if (fabsf(yout[0] - (0.5f * 1 - 1.f * 2 + 2.f * 3)) > 1e-6f || fabsf(yout[1] - (0.5f * 3 - 1.f * 5)) > 1e-6f) {
        fprintf(stderr, "conv stride-2 KAT: %g %g\n", yout[0], yout[1]); return 1;
    }

    /* 5. error behaviour: unknown variable names are rejected like assign_from_values does */
    float dummy = 0.f; int64_t shp[1] = {1};
    if (h3d_load_weight(ctx, "HandSegNet/no_such_layer/weights", &dummy, shp, 1) != H3D_EWEIGHTS) { fprintf(stderr, "unknown name accepted\n"); return 1; }

    printf("C ABI smoke OK (launches: %lld)\n", (long long)h3d_launch_count(ctx));
    h3d_destroy(ctx);
    return 0;
}

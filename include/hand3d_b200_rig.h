/* hand3d_b200 C ABI, camera rigs: h3d_resize_frames_fmt with a size and a pixel format per batch slot (DESIGN.md section 4.19).
 * Included by hand3d_b200.h, inside its declarations; not meant to be included on its own.  An entry added here is bound in
 * hand3d_b200/_lib.py's RIG_SIGNATURES and listed in tests/test_frames_rig_cpu.py's ENTRIES and in tests/test_gpu_frames_rig.py's
 * RIG_LAUNCH_CASES (its launch count against the profiler) or RIG_LAUNCH_EXCLUDED; tests/test_frames_rig_cpu.py fails otherwise. */
#ifndef HAND3D_B200_RIG_H
#define HAND3D_B200_RIG_H

/* Camera rigs: B frames of (possibly) different sizes and formats, one per batch slot, resized into one out [B,out_h,out_w,3] batch.
 * formats [B] (H3D_PIXEL_*) and hw [B,2] (H, W per slot) are host arrays; each slot obeys the pixel-format table above (the slot's index
 * is named in the refusal), 1 <= B <= H3D_FRAME_RIG_MAX_SLOTS, 1 <= out_h, out_w <= H3D_FRAME_MAX_OUT.  Slot b of out is exactly
 * h3d_resize_frames_fmt of frame b alone.
 *
 * A rig's plan is one int32 table and one int32 coefficient buffer, uploaded together into plan-owned device memory.  The table is
 * B slot records of H3D_FRAME_RIG_SLOT_WORDS words, then the order [B] (the slots grouped by format, in format order, slot index order
 * within a format), then H3D_PIXEL_YUYV + 1 launch records of H3D_FRAME_RIG_LAUNCH_WORDS words, one per format (slots == 0: no launch).
 * A slot record is its format, its picture size, the launch geometry of a single-size plan of that format and size (band: output rows
 * per CTA, nbands = ceil(out_h / band), chunk: input rows per stage, the staged row's stride and segment slots, the shared-memory
 * carve-up), the word offsets of its xb / kx / yb / ky tables in the coefficient buffer, the first CTA of its (slot, band) range within
 * its format's launch, and the index of its size among the rig's distinct sizes.  The coefficient buffer is the normalisation table
 * (256 float32 words) and then, per distinct (H, W) in order of first appearance, that size's xb [2 out_w], kx [out_w, kxs], yb
 * [2 out_h] and ky [out_h, kys], the tables h3d_resize_frames_fmt builds for it.  CTA c of format f's launch serves the slot whose
 * range holds c, band c - cta0. */
#define H3D_FRAME_RIG_MAX_SLOTS 64
#define H3D_FRAME_RIG_SLOT_WORDS 24
#define H3D_RIG_FORMAT 0
#define H3D_RIG_H 1
#define H3D_RIG_W 2
#define H3D_RIG_KXS 3
#define H3D_RIG_KYS 4
#define H3D_RIG_BAND 5
#define H3D_RIG_CHUNK 6
#define H3D_RIG_ROW_STRIDE 7
#define H3D_RIG_NBANDS 8
#define H3D_RIG_ACC_BYTES 9
#define H3D_RIG_INTER_BYTES 10
#define H3D_RIG_SMEM 11
#define H3D_RIG_SEG_OFF 12 /* 3 words: each YUV segment's slot in a staged row */
#define H3D_RIG_RGB_STRIDE 15
#define H3D_RIG_XB 16
#define H3D_RIG_KX 17
#define H3D_RIG_YB 18
#define H3D_RIG_KY 19
#define H3D_RIG_CTA0 20
#define H3D_RIG_SIZE 21 /* words 22, 23 are zero */
#define H3D_FRAME_RIG_LAUNCH_WORDS 4
#define H3D_RIG_LAUNCH_FIRST 0 /* its first position in the order */
#define H3D_RIG_LAUNCH_SLOTS 1
#define H3D_RIG_LAUNCH_CTAS 2
#define H3D_RIG_LAUNCH_SMEM 3 /* the largest of its slots' */
/* The plan of a rig on the host, without a context or a device: *table_words and *coef_words receive the sizes; table and coef (either
 * may be NULL) receive the contents when their capacities (in words, given in *table_words / *coef_words on entry when the pointer is
 * not NULL) suffice.  Refusals as h3d_resize_frames_rig's. */
H3D_API int h3d_frame_rig_query(int B, const int* formats, const int* hw, int out_h, int out_w, int32_t* table, int64_t* table_words,
                                int32_t* coef, int64_t* coef_words);
/* Builds (once per context, formats, sizes and output size) the rig's plan and uploads it on `stream`: not while `stream` is being
 * captured.  h3d_resize_frames_rig builds a missing plan itself, outside capture. */
H3D_API int h3d_frame_rig_plan(h3d_ctx* ctx, int B, const int* formats, const int* hw, int out_h, int out_w, void* stream);
/* frames: a host array of B device pointers, frame b in formats[b] at hw[b] (contiguous).  One kernel per format present (at most five),
 * each a CTA per (slot, band) of that format's slots; nothing but `out` is written.  With its plan built, it only enqueues
 * (capturable: the frame pointers travel as kernel parameters); a missing plan under capture is H3D_EINVAL. */
H3D_API int h3d_resize_frames_rig(h3d_ctx* ctx, const uint8_t* const* frames, int B, const int* formats, const int* hw, int out_h, int out_w,
                                  int normalize, void* out, void* stream);
#endif /* HAND3D_B200_RIG_H */

/*
 * fn2_flow.h -- C-ABI of libfn2.so for ground-truth flow files: the payloads of .flo, PFM and KITTI PNG files, copied to the
 * device as the bytes they hold after their header (a PNG: once the host has undone its container), converted there to a
 * network input (the input side of the reference's convert_imageset_and_flow + CustomData training path, without the
 * host-side conversions), and for the flow going out: KITTI PNG scanlines, colour-coded images and forward-backward occlusion
 * masks.  The sibling of fn2_frames.h; fn2.h, fn2_frames.h and this header together state the ABI, with
 * fn2.h's conventions: status 0 or negative with the message in fn2_last_error().
 *
 * Formats:
 *   FN2_FLOW_FLO      .flo: little-endian float [N][H][W][2], the payload after the 12-byte 'PIEH' header;
 *   FN2_FLOW_PFM      'PF' PFM with a negative scale (little-endian): float [N][H][W][3], rows stored bottom-to-top;
 *   FN2_FLOW_PFM_BE   the same with a positive scale (big-endian);
 *   FN2_FLOW_KITTI    a KITTI flow PNG's unfiltered samples: big-endian uint16 [N][H][W][3] (below).
 * A payload is 4-byte aligned in the float formats and 2-byte aligned in FN2_FLOW_KITTI.  A PFM is read top-down and keeps
 * channels 0 and 1, as the reference's CImg load_pfm + mirror('y') hands it over.
 *
 * Flag FN2_FLOW_UINT16FLOW gives the values the reference's training data holds after convert_imageset_and_flow (short(32 v),
 * NaN -> 32767) and CustomData's DecodeData (32767 -> NaN, else short / 32): t = trunc(32 v); NaN when v is NaN or t is
 * outside [-32768, 32766], else t / 32 (a t of zero gives +0).  Below -32768 the reference is undefined; here it is NaN, a
 * value the NaN-aware L1Loss and Downsample ignore.  Without the flag the floats pass through unchanged.
 *
 * KITTI flow PNGs (the KITTI 2012 / 2015 devkit's convention, readme.txt / io_flow.h): colour type 2 (RGB), bit depth 16,
 * not interlaced; R = u, G = v, B = valid as stored.  The host only undoes the PNG container: inflate, then the per-row
 * filters (fn2_png_unfilter), giving the payload [N][H][W][3] big-endian uint16, H*W*6 bytes per file.  Decode: a pixel is
 * valid when B > 0, then u = (R - 32768) / 64 and v = (G - 32768) / 64 in float32 (exact); an invalid pixel is NaN in both
 * channels, the project's marker for missing flow.  FN2_FLOW_UINT16FLOW applies the same trunc(32 v) / 32 as above.
 * Encode (the devkit's writeFlowField): a pixel is valid when both components are finite; a valid pixel stores
 * (uint16) max(min(64 v + 32768, 65535), 0) for u and v (float32, truncating) and B = 1, any other pixel (0, 0, 0).  Every
 * encoded row is filtered with Paeth (type 4): the scanline is the filter byte 4, then the 6 W filtered bytes.
 *
 * Flow colour coding (the Middlebury colour code of Baker et al., colorcode.cpp): 8-bit R, G, B per pixel.  A pixel is known
 * when both components are finite and at most 1e9 in absolute value (UNKNOWN_FLOW_THRESH, fn2_flow_error's valid ground
 * truth); an unknown pixel is (0, 0, 0).  The wheel holds 55 colours in segments RY 15, YG 6, GC 4, CB 11, BM 13, MR 6; entry
 * i of a segment of length L is, in integer arithmetic, RY (255, 255 i / L, 0), YG (255 - 255 i / L, 255, 0),
 * GC (0, 255, 255 i / L), CB (0, 255 - 255 i / L, 255), BM (255 i / L, 0, 255), MR (255, 0, 255 - 255 i / L).  Image n's
 * scale s: max_flow when it is positive, else max[n] (fallback[n] when max[n] is negative and a fallback is given), and 1 when
 * that is not positive; max[n] is normally fn2_flow_max_radius's.  In float32, without FMA contraction, for a known (u, v):
 * fx = u / s, fy = v / s; rad = sqrtf(fx fx + fy fy); a = t / pi, t the double atan2(-fy, -fx) rounded to float32 and pi
 * the float32 pi (so (1, 0) gives exactly -1); fk = (a + 1) / 2 * 54,
 * k0 = (int) fk, k1 = (k0 + 1) % 55, f = fk - k0; per channel col = (1 - f) w[k0] / 255 + f w[k1] / 255, then
 * col = 1 - rad (1 - col) when rad <= 1, else 0.75 col; the byte is (int)(255 col).
 *
 * Forward-backward consistency (Sundaram, Brox and Keutzer, ECCV 2010; this project's occlusion estimate, see DESIGN §7): with
 * fwd the flow from frame 0 to frame 1 and bwd the flow from frame 1 to frame 0, a pixel of frame 0 is occluded (255) or
 * visible (0).  For pixel (n, y, x), (fu, fv) = fwd(n, y, x):
 *   255 when fu or fv is not finite;
 *   255 when the point (x + fu, y + fv) is outside the image: FlowWarp's test x2 >= 0, y2 >= 0, x2 < W, y2 < H on the float32
 *       x2 = x + fu, y2 = y + fv;
 *   else (bu, bv) = bwd sampled there with FlowWarp's bilinear taps and mix, the values fn2_flow_warp_forward(image = bwd,
 *       flow = fwd) writes: ix = (int) x2, iy = (int) y2, ix1 = min(ix + 1, W - 1), iy1 = min(iy + 1, H - 1),
 *       a = x2 - ix, b = y2 - iy, per channel ((1-a)(1-b) TL + a(1-b) TR) + (1-a) b BL) + a b BR;
 *   255 when bu or bv is not finite (a tap that is not finite makes the sample so even at weight 0);
 *   else du = fu + bu, dv = fv + bv, lhs = du du + dv dv, mag = (fu fu + fv fv) + (bu bu + bv bv), and the pixel is 255 iff
 *       lhs > alpha1 mag + alpha2.
 * All in float32 with every product rounded separately (no FMA), in the order written, so a float32 restatement reproduces
 * every byte.  Sundaram et al. use alpha1 = 0.01, alpha2 = 0.5.  The mask of frame 1 is the same call with fwd and bwd
 * exchanged.
 */
#ifndef FN2_FLOW_H_
#define FN2_FLOW_H_

#include "fn2.h"

#define FN2_FLOW_FLO 0
#define FN2_FLOW_PFM 1
#define FN2_FLOW_PFM_BE 2
#define FN2_FLOW_KITTI 3
#define FN2_FLOW_UINT16FLOW 1

#ifdef __cplusplus
extern "C" {
#endif

/* src_dev (device payloads of dst.n files of one format, back to back, aligned as the format needs) -> dst, any float view of
 * shape (N, 2, H, W), on stream.  Writes only dst's two channels.  FN2_ERR_INVALID for an unknown format or flag, a
 * misaligned src_dev or dst.c != 2. */
FN2_API int fn2_flow_to_tensor(const void* src_dev, int format, int flags, const fn2_tensor* dst, void* stream);
/* Input blob `blob` of shape (N, 2, H, W) from device flow payloads, ordered on the net's stream. */
FN2_API int fn2_net_set_input_flow_device(fn2_net* net, const char* blob, const void* dev, int format, int flags);

/* src, any float view of shape (N, 2, H, W), 4-byte aligned -> dst_dev: N*H PNG scanlines of 1 + 6 W bytes, Paeth-filtered
 * (image n's row y at (n H + y)(1 + 6 W); the first row of every image is filtered against zeros), on stream.
 * FN2_ERR_INVALID for src.c != 2 or a misaligned src. */
FN2_API int fn2_flow_to_kitti_png_rows(const fn2_tensor* src, void* dst_dev, void* stream);
/* src, any float view of shape (N, 2, H, W), 4-byte aligned -> max_dev[n] (N floats, 4-byte aligned): the largest float32
 * sqrtf(u u + v v) over image n's known pixels, -1 for an image without one; on stream, no host synchronisation.  Exact (a
 * maximum).  FN2_ERR_INVALID for src.c != 2, N above 65535 or a misaligned pointer. */
FN2_API int fn2_flow_max_radius(const fn2_tensor* src, float* max_dev, void* stream);
/* src, any float view of shape (N, 2, H, W), 4-byte aligned -> dst_dev: the colour code above as dense [N][H][W][3] bytes
 * (R, G, B), on stream.  Scale: max_flow > 0, or max_flow = 0 with max_dev (N floats on the device, 4-byte aligned) and
 * optionally fallback_dev (the same, or null).  FN2_ERR_INVALID for src.c != 2, a misaligned pointer, a max_flow that is
 * negative or not finite, and max_flow = 0 without max_dev. */
FN2_API int fn2_flow_to_color(const fn2_tensor* src, const float* max_dev, const float* fallback_dev, float max_flow, void* dst_dev,
                              void* stream);
/* As fn2_flow_to_color, written as N*H PNG scanlines of 1 + 3 W bytes for 8-bit RGB (colour type 2, bit depth 8),
 * Paeth-filtered with 3 bytes per pixel (image n's row y at (n H + y)(1 + 3 W); the first row of every image is filtered against
 * zeros), the row layout of fn2_flow_to_kitti_png_rows. */
FN2_API int fn2_flow_to_color_png_rows(const fn2_tensor* src, const float* max_dev, const float* fallback_dev, float max_flow,
                                       void* dst_dev, void* stream);
/* fwd, bwd: float views of one shape (N, 2, H, W), any strides, 4-byte aligned -> frame 0's occlusion mask by the
 * forward-backward check above, one byte per pixel: pixel (n, y, x) at out_dev + n pair_stride + y row_stride + x, on stream.
 * Nothing else of out_dev is written, so row_stride = 1 + W with out_dev one byte into a buffer gives PNG scanlines of
 * 8-bit grey (filter None where the buffer holds zeros).  FN2_ERR_INVALID for shapes that differ, c != 2, an alpha that is
 * negative or not finite, row_stride < W, pair_stride < H row_stride, N above 65535 (the grid's limit) or a misaligned flow. */
FN2_API int fn2_flow_fb_occlusion(const fn2_tensor* fwd, const fn2_tensor* bwd, float alpha1, float alpha2, void* out_dev,
                                  size_t row_stride, size_t pair_stride, void* stream);
/* Host: undoes PNG's per-row filters (types 0-4) of `rows` scanlines of 1 + row_bytes bytes at src into rows * row_bytes
 * bytes at dst; bpp: bytes per complete pixel (1..8), the filters' left distance.  The first row is filtered against zeros.
 * FN2_ERR_INVALID for a filter type above 4, naming the row.  No device work. */
FN2_API int fn2_png_unfilter(const void* src, int rows, size_t row_bytes, int bpp, void* dst);

#ifdef __cplusplus
}
#endif

#endif /* FN2_FLOW_H_ */

/*
 * fn2_flow.h -- C-ABI of libfn2.so for ground-truth flow files: the payloads of .flo and PFM files, copied to the device as
 * the bytes they hold after their header, converted there to a network input (the input side of the reference's
 * convert_imageset_and_flow + CustomData training path, without the host-side conversions).  The sibling of fn2_frames.h;
 * fn2.h, fn2_frames.h and this header together state the ABI, with fn2.h's conventions: status 0 or negative with the message
 * in fn2_last_error().
 *
 * Formats:
 *   FN2_FLOW_FLO      .flo: little-endian float [N][H][W][2], the payload after the 12-byte 'PIEH' header;
 *   FN2_FLOW_PFM      'PF' PFM with a negative scale (little-endian): float [N][H][W][3], rows stored bottom-to-top;
 *   FN2_FLOW_PFM_BE   the same with a positive scale (big-endian).
 * A PFM is read top-down and keeps channels 0 and 1, as the reference's CImg load_pfm + mirror('y') hands it over.
 *
 * Flag FN2_FLOW_UINT16FLOW gives the values the reference's training data holds after convert_imageset_and_flow (short(32 v),
 * NaN -> 32767) and CustomData's DecodeData (32767 -> NaN, else short / 32): t = trunc(32 v); NaN when v is NaN or t is
 * outside [-32768, 32766], else t / 32 (a t of zero gives +0).  Below -32768 the reference is undefined; here it is NaN, a
 * value the NaN-aware L1Loss and Downsample ignore.  Without the flag the floats pass through unchanged.
 */
#ifndef FN2_FLOW_H_
#define FN2_FLOW_H_

#include "fn2.h"

#define FN2_FLOW_FLO 0
#define FN2_FLOW_PFM 1
#define FN2_FLOW_PFM_BE 2
#define FN2_FLOW_UINT16FLOW 1

#ifdef __cplusplus
extern "C" {
#endif

/* src_dev (device payloads of dst.n files, back to back, 4-byte aligned) -> dst, any float view of shape (N, 2, H, W), on
 * stream.  Writes only dst's two channels.  FN2_ERR_INVALID for an unknown format or flag, a misaligned src_dev or
 * dst.c != 2. */
FN2_API int fn2_flow_to_tensor(const void* src_dev, int format, int flags, const fn2_tensor* dst, void* stream);
/* Input blob `blob` of shape (N, 2, H, W) from device flow payloads, ordered on the net's stream. */
FN2_API int fn2_net_set_input_flow_device(fn2_net* net, const char* blob, const void* dev, int format, int flags);

#ifdef __cplusplus
}
#endif

#endif /* FN2_FLOW_H_ */

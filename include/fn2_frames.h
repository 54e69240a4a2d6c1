/*
 * fn2_frames.h -- C-ABI of libfn2.so for 8-bit image frames: frames converted to a network input on the device, and blobs
 * read back channel-fast (scripts/run-flownet.py:30-35 and :98-126 of the reference, without the host-side conversions).
 * fn2.h and this header together state the ABI; the conventions are fn2.h's: status 0 or negative with the message in
 * fn2_last_error().
 *
 * Frames are dense bytes [N][H][W][K], K = 1 (gray), 3 (RGB) or 4 (RGBA; alpha is ignored).  They become the float blob
 * channels 0, 1, 2 = B, G, R with values 0..255, exactly as image_to_blob's floats; a gray frame fills all three channels,
 * as pycaffe broadcasts the (1, 1, H, W) array the reference builds for it (python/caffe/pycaffe.py:119).
 */
#ifndef FN2_FRAMES_H_
#define FN2_FRAMES_H_

#include "fn2.h"

#ifdef __cplusplus
extern "C" {
#endif

/* frames_dev (device bytes [dst.n][dst.h][dst.w][channels]) -> dst, any float view of shape (N, 3, H, W), on stream.  Writes
 * only dst's three channels.  FN2_ERR_INVALID for channels not in {1, 3, 4} or dst.c != 3. */
FN2_API int fn2_frames_to_tensor(const void* frames_dev, int channels, const fn2_tensor* dst, void* stream);
/* Input blob `blob` of shape (N, 3, H, W) from host frames [N][H][W][channels]: the bytes go to the net's staging buffer
 * (H2D), then fn2_frames_to_tensor; asynchronous on the net's stream like fn2_net_set_input (host_frames must stay valid
 * until the stream has run the copy). */
FN2_API int fn2_net_set_input_frames(fn2_net* net, const char* blob, const void* host_frames, int channels);
/* The same from device frames, ordered on the net's stream. */
FN2_API int fn2_net_set_input_frames_device(fn2_net* net, const char* blob, const void* dev_frames, int channels);
/* Blob as dense NHWC floats (for the flow: the payload order of a .flo file).  The host variant synchronises the net's
 * stream like fn2_net_get_blob; the device variant is asynchronous on it. */
FN2_API int fn2_net_get_blob_nhwc(fn2_net* net, const char* blob, float* host);
FN2_API int fn2_net_get_blob_nhwc_device(fn2_net* net, const char* blob, float* dev);

#ifdef __cplusplus
}
#endif

#endif /* FN2_FRAMES_H_ */

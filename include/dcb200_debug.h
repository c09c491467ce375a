/* dcb200 -- developer / test hooks of libdcb200.so.  NOT part of the drop-in boundary (include/dcb200.h): nothing a
 * caller of the model path needs.  Used by tests/ and scripts/ to look inside a forward pass. */
#ifndef DCB200_DEBUG_H_
#define DCB200_DEBUG_H_

#include "dcb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Debug/test hook: copy the fp32 residual stream after stage `stage` of the LAST chunk of the
 * last forward into out [tokens, 280] (row-major).  stage 0 = condenser+pos-enc,
 * 1+2n = attention sub-layer n, 2+2n = FFN sub-layer n.  Requires dcb_set_debug(e, 1). */
int dcb_set_debug(dcb_engine* e, int32_t enabled);
int dcb_debug_residual(dcb_engine* e, int32_t stage, float* out, int64_t out_elems);

/* Debug/test hook: copy bf16 operand image `which` as captured at stage `stage` (numbered as for
 * dcb_debug_residual) of the LAST chunk of the last forward into out [tokens, width] as raw bf16 bits,
 * token-major, at the image's full padded width (padding columns included):
 *   DCB_DEBUG_EMBED  stage 0       the concatenated embeddings (width = E rounded up to 16)
 *   DCB_DEBUG_XB     stage 0       layer 0's q/k/v operand (288)
 *                    stage 1+2n    layer n's FFN operand (288)
 *                    stage 2+2n    layer n+1's q/k/v operand (288; not after the last layer)
 *   DCB_DEBUG_QKV    stage 1+2n    q/k/v of layer n (864: q_h0 q_h1 k_h0 k_h1 v_h0 v_h1, 144 each)
 *   DCB_DEBUG_ATT    stage 1+2n    attention output of layer n (288: two heads of 144)
 *   DCB_DEBUG_HID    stage 2+2n    ReLU hidden activation of layer n (filter_size)
 * Capture is a stream-ordered device copy at the same points as the residual's.  Requires
 * dcb_set_debug(e, 1). */
enum { DCB_DEBUG_EMBED = 0, DCB_DEBUG_XB = 1, DCB_DEBUG_QKV = 2, DCB_DEBUG_ATT = 3, DCB_DEBUG_HID = 4 };
int dcb_debug_operand(dcb_engine* e, int32_t stage, int32_t which, uint16_t* out, int64_t out_elems);

/* Debug/test hook: copy float32 image `which` as captured at stage `stage` (numbered as for dcb_debug_residual) of
 * the LAST chunk of the last float32 forward (strict fp32 or tf32x3) into out [tokens, width], row-major:
 *   DCB_DEBUG_F32_EMB  stage 0             the concatenated embeddings (width E, unpadded)
 *   DCB_DEBUG_F32_X    every stage         the residual after the stage (280)
 *   DCB_DEBUG_F32_Y    stages 1+2n, 2+2n   the LayerNorm output the stage's GEMMs read (280; pre-LN models only)
 *   DCB_DEBUG_F32_Q, _K, _V, _ATT
 *                      stage 1+2n          q (scaled by depth^-1/2), k, v and the attention output of layer n (280)
 *   DCB_DEBUG_F32_HID  stage 2+2n          ReLU hidden activation of layer n (filter_size)
 * Capture is a stream-ordered device copy after the launches that wrote the image, into a buffer allocated on the
 * first float32 forward with dcb_set_debug(e, 1) and freed by dcb_set_debug(e, 0).  DCB_ERR_STATE without capture or
 * before such a forward; DCB_ERR_INVALID for a pair not captured or an output too small. */
enum {
  DCB_DEBUG_F32_EMB = 0, DCB_DEBUG_F32_X = 1, DCB_DEBUG_F32_Y = 2, DCB_DEBUG_F32_Q = 3, DCB_DEBUG_F32_K = 4,
  DCB_DEBUG_F32_V = 5, DCB_DEBUG_F32_ATT = 6, DCB_DEBUG_F32_HID = 7
};
int dcb_debug_f32(dcb_engine* e, int32_t stage, int32_t which, float* out, int64_t out_elems);

/* Debug/test hook: the model head's per-token epilogue (softmax, argmax, Phred, calibration, cap, round, ASCII) on
 * caller-supplied final logits, one token per row: logits [n, 5] float32 -> bases [n] (' ATCG'), quals [n]
 * (Phred+33) and probs [n, 5] (nullable), all host arrays.  The logits are taken as they are: no fc1 bias is added
 * (the epilogue runs with a zero bias).  Uses the engine's calibration and max_base_quality; needs no forward and no
 * dcb_set_debug.  Any n >= 0 (processed in chunks through device scratch).  DCB_ERR_INVALID for a null pointer or
 * n < 0. */
int dcb_debug_head_epilogue(dcb_engine* e, const float* logits, int64_t n, uint8_t* bases, uint8_t* quals, float* probs);

#ifdef __cplusplus
}
#endif
#endif /* DCB200_DEBUG_H_ */

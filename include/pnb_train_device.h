/*
 * pnb_train_device.h -- C-ABI of the trainer's forward and backward with the loss left to the caller: the two device
 * calls a torch autograd function makes (percepnet_b200/torch_module.py).  Part of the percepnet_b200.h ABI, which
 * includes this header at its end; it may also be included on its own.  Same conventions: plain pointers and sizes,
 * PNB_OK (0) or a negative error code, pnb_last_error() for the text.
 */
#ifndef PNB_TRAIN_DEVICE_H
#define PNB_TRAIN_DEVICE_H

#include <stddef.h>
#include "percepnet_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The trainer's forward and backward with the loss left to the caller (PNB_TRAIN_NETWORK engines; what a torch
 * autograd function calls, so that any loss and any optimizer train the network): the forward and the backward
 * recurrences of pnb_train_grad_*, cut where its loss sits.  Device memory only; both asynchronous on cuda_stream and
 * ordered like a call.
 *   pnb_train_forward_device  d_x holds the active rows [0, n) of network input, x_stride >= n_frames * 70: features as
 *                     rnn_train.py's model receives them (PNB_RNN_FEATURES, no x30 on the device); every row runs all
 *                     n_frames hops from zero state.  d_weights: NULL, or the N = 7 962 564 parameters in PNBW blob order
 *                     (as pnb_train_import takes them), copied into the engine's weights on cuda_stream before the
 *                     forward runs.  d_out receives g, r per hop (out_stride >= n_frames * 68) exactly as the trainer's
 *                     forward computes them (exact tanh / sigmoid, not the tansig table).  The forward's activations are
 *                     kept for its backward, and the PNB_TAP_TRAIN_FC / _C1 / _C2PRE taps show them.
 *   pnb_train_backward_device  the backward of the last forward (its n, n_frames and weights): d_dout holds dL/d(out) in
 *                     the layout of d_out (dout_stride >= n_frames * 68).  The output layers are seeded with
 *                     dout (1 - p) p evaluated left to right in fp32 (ATen's sigmoid_backward, so the same bits torch's
 *                     autograd would pass there; PNB_TAP_TRAIN_DPRE shows them).  d_dx: NULL, or dL/dx in the layout of
 *                     d_x (dx_stride >= n_frames * 70).  The parameter gradient becomes the engine's held gradient, as
 *                     after pnb_train_grad_* with n x n_frames counted hops (pnb_train_adam / _accumulate use it), and
 *                     d_grad, when not NULL, receives it in blob order (N floats).  A non-finite value in it skips the next
 *                     pnb_train_adam on the device but does not raise PNB_ERR_DOMAIN: the caller owns the loss, and
 *                     non-finite gradients pass through as torch passes them.
 * A forward waits for one backward; pnb_reset, pnb_set_active_streams, a pnb_train_grad_* call, pnb_train_adam,
 * pnb_train_import of PNB_TRAIN_WEIGHTS (the last two rewrite the weights the backward would take) and that backward
 * end the wait; imports of the moments or the accumulator, pnb_train_accumulate and pnb_train_finish keep it.
 * Refused with PNB_ERR_ARG before anything is enqueued: an engine without PNB_TRAIN_NETWORK, n_frames outside
 * [1, max_frames_per_call], a NULL d_x, d_out or d_dout, a short stride, a backward with no forward waiting for it, a
 * poisoned engine (PNB_ERR_CUDA).  Each call issues a fixed number of launches whatever n_frames: 17 for a forward,
 * 100 for a backward, 102 with d_dx. */
int pnb_train_forward_device(pnb_engine *e, const float *d_x, size_t x_stride, int n_frames, const float *d_weights,
                             float *d_out, size_t out_stride, void *cuda_stream);
int pnb_train_backward_device(pnb_engine *e, const float *d_dout, size_t dout_stride, float *d_dx, size_t dx_stride,
                              float *d_grad, void *cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* PNB_TRAIN_DEVICE_H */

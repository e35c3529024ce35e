/*
 * pnb_train_state.h -- C-ABI of the trainer's forward and backward with network state carried in and out and windows
 * of their own lengths: what truncated backpropagation through time over consecutive windows of one stream calls
 * (percepnet_b200/torch_module.py).  Part of the percepnet_b200.h ABI, which includes this header at its end; it may also
 * be included on its own.  Same conventions: plain pointers and sizes, PNB_OK (0) or a negative error code,
 * pnb_last_error() for the text.
 */
#ifndef PNB_TRAIN_STATE_H
#define PNB_TRAIN_STATE_H

#include <stddef.h>
#include "percepnet_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The network state of one window, in floats:
 *   [fc_hist 4 x 128][c1_hist 2 x 512][gru1 512][gru2 512][gru3 512][gru_gb 512][gru_rb 128]
 * fc_hist: the last four fc outputs (after ReLU, oldest first), conv1's input history; c1_hist: the last two conv1
 * outputs (after ReLU, oldest first), conv2's input history; then the five GRU states.  The same order as a stream
 * state's network part (bytes 39 736 to 54 583 of a pnb_get_state blob).  A forward from state S over hops [0, T) is
 * rnn_train.py's PercepNet run on the hops that produced S followed by these T hops; zero state is a window's start. */
#define PNB_TRAIN_STATE_FLOATS 3712

/* pnb_train_forward_device and pnb_train_backward_device (pnb_train_device.h) with state; those two are these with every
 * state array and lengths NULL, the same bits and the same launches.  Device memory only but lengths; asynchronous on
 * cuda_stream and ordered like a call.
 *   pnb_train_forward_state_device  lengths: NULL (every window runs n_frames hops), or a host array of one count in
 *                     [1, n_frames] per active row, read before the call returns: window b's input past hop lengths[b]
 *                     is ignored, its d_out rows there are written as zeros, and the held gradient of its backward
 *                     counts sum(lengths) hops.  d_state_in: NULL (zero state), or one state row per active window
 *                     (state_in_stride >= PNB_TRAIN_STATE_FLOATS) that the window starts from.  d_state_out: NULL, or
 *                     rows (state_out_stride >= PNB_TRAIN_STATE_FLOATS) that receive each window's state after its last
 *                     hop, lengths[b] (a window shorter than four hops passes part of its state in through).  The rest
 *                     as pnb_train_forward_device.
 *   pnb_train_backward_state_device  the backward of the last forward: d_dstate_out: NULL (no gradient at the state
 *                     out), or dL/d(state out) in the layout of d_state_out.  d_dstate_in: NULL, or rows that receive
 *                     dL/d(state in), whether or not that forward had a state in (without one, the gradient at its zero
 *                     state).  The rest as pnb_train_backward_device; hops past a window's end take no gradient, whatever
 *                     d_dout holds there.
 * Refused with PNB_ERR_ARG before anything is enqueued: everything pnb_train_*_device refuses, a length outside
 * [1, n_frames], a short state stride.  Each call issues a fixed number of launches whatever n_frames:
 *   forward   17, + 1 with d_state_in, + 2 with lengths, + 1 with d_state_out
 *   backward 100, + 2 with d_dx, + 1 with d_dstate_out, + 6 with d_dstate_in */
int pnb_train_forward_state_device(pnb_engine *e, const float *d_x, size_t x_stride, int n_frames, const int *lengths,
                                   const float *d_weights, const float *d_state_in, size_t state_in_stride,
                                   float *d_out, size_t out_stride, float *d_state_out, size_t state_out_stride,
                                   void *cuda_stream);
int pnb_train_backward_state_device(pnb_engine *e, const float *d_dout, size_t dout_stride,
                                    const float *d_dstate_out, size_t dstate_out_stride, float *d_dx, size_t dx_stride,
                                    float *d_dstate_in, size_t dstate_in_stride, float *d_grad, void *cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* PNB_TRAIN_STATE_H */

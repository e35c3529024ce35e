/*
 * pnb_synth_grad.h -- C-ABI of the synthesis's gradient: dL/d(g, r) of a loss on the PCM that pnb_synthesize_* writes,
 * so that the gain network trains on the enhanced waveform (percepnet_b200/torch_signal.py).  Part of the
 * percepnet_b200.h ABI, which includes this header at its end; it may also be included on its own.  Same conventions:
 * plain pointers and sizes, PNB_OK (0) or a negative error code, pnb_last_error() for the text.  Device memory only,
 * asynchronous on cuda_stream.
 */
#ifndef PNB_SYNTH_GRAD_H
#define PNB_SYNTH_GRAD_H

#include <stddef.h>
#include "percepnet_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The synthesis operands of one hop, in floats: everything the synthesis of that hop reads but g/r and the overlap-add
 * memory.
 *   [0, 800)      X, bins 0..399 (re, im interleaved): the spectrum the synthesis reads from the ring slot of hop c - 5
 *   [800, 1600)   P, bins 0..399: the comb-filtered spectrum
 *   [1600, 1634)  the band energies the post-filter weighs (PNB_TAP_EX of the hop)
 *   [1634]        the silence flag, 0.0 or 1.0
 *   [1635]        0, so that every hop starts on a 16-byte boundary */
#define PNB_SYNTH_OPS_FLOATS 1636

/* pnb_synthesis_operands_device: the operands of the pending synthesis (the last pnb_analyze_*) of the active rows
 * [0, n), its F hops: row i receives F x PNB_SYNTH_OPS_FLOATS floats, ops_stride >= F * PNB_SYNTH_OPS_FLOATS.  They are
 * read at the addresses the synthesis kernel reads, the spectra of earlier calls included, so they are the synthesis's
 * operands by construction.  It touches no signal state and leaves the synthesis pending; one launch, ordered like a
 * call.  PCM engines (fp32 or tensor, PNB_CONV_WIDE and PNB_POSTFILTER included) and PNB_SIGNAL_ONLY engines, slot mode.
 * Refused with PNB_ERR_ARG before anything is enqueued: nothing pending, an engine in session mode, PNB_NETWORK_ONLY,
 * PNB_TRAIN_NETWORK and PNB_TRAIN_DATA engines, d_ops NULL, a short stride; a poisoned engine returns PNB_ERR_CUDA. */
int pnb_synthesis_operands_device(pnb_engine *e, float *d_ops, size_t ops_stride, void *cuda_stream);

/* pnb_synthesis_backward_device: dL/d(g, r) from dL/d(out) for n_rows rows of n_frames hops; needs no engine, only the
 * operands (pnb_synthesis_operands_device) and the g/r that synthesis took.  postfilter: 0 or 1, the PNB_POSTFILTER
 * setting of the engine that synthesised (the gradient then passes through the envelope post-filter).
 *   d_ops    rows of n_frames x PNB_SYNTH_OPS_FLOATS, ops_stride >= n_frames * PNB_SYNTH_OPS_FLOATS
 *   d_gr     rows of n_frames x 68 (34 g then 34 r per hop) as pnb_synthesize_* took them, gr_stride >= n_frames * 68
 *   d_dout   rows of n_frames x 480, dL/d(out) of the f32 PCM the synthesis wrote, dout_stride >= n_frames * 480
 *   d_dgr    rows of n_frames x 68 that receive dL/d(g, r), dgr_stride >= n_frames * 68
 * Out hop t is the first half of hop t's windowed inverse transform plus the second half of hop t - 1's, so dL/d(g, r)
 * of hop t depends on dL/d(out) of hops t and t + 1.  The second half of the last hop goes to the overlap-add memory the
 * call leaves for the next call and takes no gradient: the graph is cut at the call's edge.  There is no gradient with
 * respect to the PCM input (the pitch search and the silence decision are not differentiable).  On a silent hop dL/dr
 * is exactly 0; with the post-filter, a hop whose 34 g are all zero (where the filtered gains vanish to second order)
 * gets exactly 0 for dL/dg.  For non-finite g/r or dL/d(out) the affected row's gradient is unspecified and the other
 * rows are unaffected.  One launch, asynchronous on cuda_stream, current device.
 * Refused with PNB_ERR_ARG before anything is enqueued: a NULL pointer, a short stride, n_rows < 1, n_frames < 1,
 * postfilter other than 0 or 1. */
int pnb_synthesis_backward_device(const float *d_ops, size_t ops_stride, const float *d_gr, size_t gr_stride,
                                  long long n_rows, int n_frames, int postfilter, const float *d_dout,
                                  size_t dout_stride, float *d_dgr, size_t dgr_stride, void *cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* PNB_SYNTH_GRAD_H */

#!/usr/bin/env python
"""Launch timeline of two submitted long calls: prints every launch with its start/end and the busy time of the network
and DSP kernels.  Run on the GPU box: python tools/timeline.py [streams] [frames]."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.weights import synth_model  # noqa: E402
from bench import make_step_inputs  # noqa: E402


def main():
    S = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    F = int(sys.argv[2]) if len(sys.argv) > 2 else 100
    dev = torch.device("cuda", 0)
    eng = api.Engine(S, F, synth_model(0), api.NN_TENSOR)
    bufs = make_step_inputs(S, F, 2, 0, dev)
    outs = [torch.empty_like(b) for b in bufs]
    st = torch.cuda.current_stream()
    for i in range(3):
        eng.process_device(bufs[i % 2].data_ptr(), bufs[i % 2].stride(0), outs[i % 2].data_ptr(), outs[i % 2].stride(0), F, stream=st.cuda_stream)
    torch.cuda.synchronize()
    eng.profile(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for i in range(2):
        eng.submit_device(bufs[i].data_ptr(), bufs[i].stride(0), outs[i].data_ptr(), outs[i].stride(0), F, stream=st.cuda_stream)
    eng.flush(st.cuda_stream)
    e1.record(st)
    torch.cuda.synchronize()
    tl = eng.profile_timeline()
    eng.profile(False)
    net = {"tc_gemm_kernel", "tc_aux_kernel"}
    rows = [{"k": k, "t0": round(a, 3), "t1": round(b, 3), "part": "net" if k in net else "dsp"} for k, a, b in tl]
    busy = {"net": sum(r["t1"] - r["t0"] for r in rows if r["part"] == "net"), "dsp": sum(r["t1"] - r["t0"] for r in rows if r["part"] == "dsp")}
    print(json.dumps({"two_calls_ms": e0.elapsed_time(e1), "span_ms": max(r["t1"] for r in rows), "busy_ms": busy, "launches": rows}))
    eng.close()


if __name__ == "__main__":
    main()

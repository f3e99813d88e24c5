"""Full-size synthetic traces generated on the device, for the benchmark tools and the full-size GPU tests."""


def device_traces(specs, pv0, seed_of, dev):
    """the traces of chips with fields h, g, wp, extra, extra_prep generated on the device by synth_air's torch generator (chip i from
    seed_of(i)) -> (main traces back to back, preprocessed tables back to back or None, their rows, their columns)"""
    import torch
    from sp1_b200 import synth_air as SA
    mains, preps = [], []
    for i, sp in enumerate(specs):
        m, p = SA.synth_trace_cuda(sp.h, sp.g, sp.wp, pv0, seed_of(i), dev, extra_cols=sp.extra, extra_prep=sp.extra_prep)
        mains.append(m)
        if sp.wp:
            preps.append(p)
    d_main = torch.cat(mains).contiguous()
    d_prep = torch.cat(preps).contiguous() if preps else None
    del mains, preps
    # the library reads the traces on its own stream: torch's kernels that wrote them must have finished
    torch.cuda.current_stream(dev).synchronize()
    return d_main, d_prep, [sp.h for sp in specs if sp.wp], [1 + sp.extra_prep for sp in specs if sp.wp]

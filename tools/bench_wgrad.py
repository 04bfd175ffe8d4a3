"""GPU: per-layer time of the TF32 conv weight gradient (avc_conv_wgrad_tc: the MMA kernel plus its slice reduction) at
the shapes of one training step.

    python tools/bench_wgrad.py [--batch 256] [--seg 128] [--c-in 80 512] [--json FILE]

The descriptors are recorded from one eager training step of the engine on the real library (every weight-gradient
launch of the step, in order), then every distinct descriptor is timed on its own: a CUDA graph of --reps launches,
each with its own operand set, rotating over enough sets that the operands exceed the 50 MB L2, timed with CUDA events
after a warm-up replay.  FLOPs are the algorithmic 2 B Tout Cin Cout K of the shape; the TF32 share is of the H100 SXM
data-sheet rate (495 TFLOP/s dense at 700 W), which a power-limited card does not reach.  The card, its power limit and
SM clock are printed with the table.
"""
import argparse
import ctypes as C
import itertools
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from _harness import card, graph_us  # noqa: E402

TF32_PEAK = 495.0     # TFLOP/s, H100 SXM data sheet, dense, 700 W
L2_BYTES = 50 << 20


class Recorder:
    """The engine's library with the weight-gradient entry points recording their descriptors."""

    def __init__(self, real):
        self.real, self.descs = real, []

    def __getattr__(self, name):
        return getattr(self.real, name)

    def _rec(self, kernel, dref):
        from adaptive_voice_conversion_b200 import _lib as L
        self.descs.append((kernel, L.WgradDesc.from_buffer_copy(dref._obj)))

    def avc_conv_wgrad_tc(self, dref, *a):
        self._rec("tc", dref)
        return self.real.avc_conv_wgrad_tc(dref, *a)

    def avc_conv_wgrad_tc_acc(self, dref, *a):
        self._rec("tc", dref)
        return self.real.avc_conv_wgrad_tc_acc(dref, *a)

    def avc_conv_wgrad(self, dref, *a):
        self._rec("simt", dref)
        return self.real.avc_conv_wgrad(dref, *a)


def step_descriptors(c_in, B, T, dev):
    """(kernel, descriptor) of every weight-gradient launch of one eager training step."""
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.engine import A4, Engine
    cfg = orc.default_config(c_in)
    e = Engine(cfg, dev)
    e.precision = "tf32"
    P = {k: v.to(dev) for k, v in orc.init_state(cfg, seed=0).items()}
    e.pack_weights(P, need_dgrad=True)
    e.lib = Recorder(e.lib)
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    x = torch.randn(B, c_in, T, device=dev)
    emb, cs = e.speaker_fwd(P, x, True)
    mu4, ls4, ce = e.content_fwd(P, x, True)
    eps = torch.randn(B, mu4.C, mu4.T, device=dev)
    mu, ls, z4 = e.reparam_fwd(mu4, ls4, eps)
    dec4, cd = e.decoder_fwd(P, z4, emb, True)
    dy = A4.empty(dec4.B, dec4.C, dec4.T, dev)
    dy.t.normal_()
    dz4, demb = e.decoder_bwd(P, G, cd, dy)
    dmu4, dls4 = e.reparam_bwd(dz4, ls4, eps, torch.zeros_like(mu), torch.zeros_like(ls))
    e.content_bwd(P, G, ce, dmu4, dls4)
    e.speaker_bwd(P, G, cs, demb)
    torch.cuda.synchronize(dev)
    e.check_tc_status()
    return e, e.lib.descs


def layer_class(d, c_in):
    if d.Cin == c_in and d.Cout == 128 and d.stride == 1:
        return f"bank k{d.K}"
    if d.K == 1 and d.Cin > 512:
        return "in_conv"
    if d.K == 1:
        return f"k1 {d.Cin}->{d.Cout}"
    return f"{d.Cin}->{d.Cout} k{d.K}" + (" s2" if d.stride == 2 else "")


def shape_key(d):
    return (d.B, d.Cin, d.Cout, d.K, d.Tin, d.Tout, d.stride, d.pad_left, d.x_bstride, d.dc_bstride)


def time_descriptor(e, d, dev, reps):
    """Microseconds per avc_conv_wgrad_tc call (MMA kernel + reduction) on rotating operand sets."""
    from adaptive_voice_conversion_b200 import _lib as L
    lib = e.lib.real if isinstance(e.lib, Recorder) else e.lib
    nx, ndc = d.B * d.x_bstride, d.B * d.dc_bstride
    nset = max(2, min(reps, -(-2 * L2_BYTES // (4 * (nx + ndc)))))
    xs = [torch.randn(nx, device=dev) for _ in range(nset)]
    dcs = [torch.randn(ndc, device=dev) for _ in range(nset)]
    dw = torch.zeros(d.Cout * d.Cin * d.K, device=dev)
    scratch = torch.empty(int(lib.avc_wgrad_tc_scratch_floats(C.byref(d))), device=dev)
    descs = []
    for i in range(nset):
        q = L.WgradDesc.from_buffer_copy(d)
        q.x, q.dc, q.dw = xs[i].data_ptr(), dcs[i].data_ptr(), dw.data_ptr()
        descs.append(q)
    n = itertools.count()

    def launch():
        e._ck(lib.avc_conv_wgrad_tc(C.byref(descs[next(n) % nset]), scratch.data_ptr(), e.tc_status.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream), "avc_conv_wgrad_tc")
    launch()
    launch()
    us = graph_us(launch, reps, 5)
    e.check_tc_status()
    return us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seg", type=int, default=128)
    ap.add_argument("--c-in", type=int, nargs="+", default=[80, 512])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    result = {"card": card(dev), "configs": {}}
    print(f"card: {result['card']}")
    for c_in in args.c_in:
        e, launches = step_descriptors(c_in, args.batch, args.seg, dev)
        count, first = {}, {}
        for kernel, d in launches:
            if kernel != "tc":
                continue
            k = shape_key(d)
            count[k] = count.get(k, 0) + 1
            first.setdefault(k, d)
        rows, total_us, total_flop = [], 0.0, 0.0
        for k, d in first.items():
            us = time_descriptor(e, d, dev, args.reps)
            flop = 2.0 * d.B * d.Tout * d.Cin * d.Cout * d.K
            tf = flop / us / 1e6
            rows.append({"class": layer_class(d, c_in), "shape": f"B{d.B} {d.Cin}->{d.Cout} k{d.K} s{d.stride} Tout{d.Tout}",
                         "per_step": count[k], "us": us, "gflop": flop / 1e9, "tflops": tf, "tf32_share": tf / TF32_PEAK})
            total_us += us * count[k]
            total_flop += flop * count[k]
        n_simt = sum(1 for kern, _ in launches if kern != "tc")
        print(f"\nc_in = {c_in}, B = {args.batch}, segment = {args.seg}: {len(launches)} weight-gradient launches per step "
              f"({n_simt} on the FFMA kernel, not timed here)")
        print(f"{'class':18s} {'shape':36s} {'/step':>5s} {'us':>8s} {'GFLOP':>7s} {'TFLOP/s':>8s} {'of 495':>7s}")
        for r in rows:
            print(f"{r['class']:18s} {r['shape']:36s} {r['per_step']:5d} {r['us']:8.1f} {r['gflop']:7.2f} {r['tflops']:8.1f} {100 * r['tf32_share']:6.1f}%")
        print(f"{'sum over the step':18s} {'':36s} {sum(count.values()):5d} {total_us:8.1f} {total_flop / 1e9:7.2f} "
              f"{total_flop / total_us / 1e6:8.1f} {100 * total_flop / total_us / 1e6 / TF32_PEAK:6.1f}%")
        result["configs"][str(c_in)] = {"rows": rows, "step_us": total_us, "step_gflop": total_flop / 1e9}
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

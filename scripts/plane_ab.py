"""Dev probe: per-shape tap-GEMM times of HiFi-GAN V1 with and without operand-plane feed (AGPT_PLANE_FEED), two
engines in one process, minimum over profiled forwards.  Usage: python scripts/plane_ab.py [B T reps]"""
import ctypes
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from audiogpt_b200 import _lib, specs  # noqa: E402
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
T = int(sys.argv[2]) if len(sys.argv) > 2 else 800
REPS = int(sys.argv[3]) if len(sys.argv) > 3 else 3


def make(plane):
    os.environ["AGPT_PLANE_FEED"] = "1" if plane else "0"
    m = HifiGanGenerator(specs.HIFIGAN_V1)
    m.load_state_dict(specs.synth_hifigan(specs.HIFIGAN_V1, 1234))
    m = m.eval().cuda()
    m(torch.zeros(1, 80, 2, device="cuda"))
    return m


def shapes(m, mel):
    """{(kind, C, taps): ms summed over the launches of that class}, minimum per class over REPS forwards."""
    L = _lib.lib()
    best = None
    for _ in range(REPS):
        _lib.check(L.agpt_profile_enable(1))
        m(mel)
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 20)
        L.agpt_profile_dump(buf, 1 << 20)
        _lib.check(L.agpt_profile_enable(0))
        acc = defaultdict(float)
        for line in buf.value.decode().splitlines():
            v, G, Lr, cin, cout, ntaps, span, epi, wr, ms, fl = line.split()
            kind = "pair" if int(epi) >= 16 else "conv"
            acc[(kind, int(cin), int(cout), int(ntaps))] += float(ms)
        best = acc if best is None else {k: min(best[k], acc[k]) for k in acc}
    return best


mel = specs.synth_tensor((B, 80, T), seed=0, scale=2.0, shift=-4.0).cuda()
ref, pl = make(False), make(True)
for m in (ref, pl):
    for _ in range(2):
        m(mel)
torch.cuda.synchronize()
a, b = shapes(ref, mel), shapes(pl, mel)
print(f"HiFi-GAN V1 {B} x {T}: tap-GEMM ms per shape class, transform -> plane-fed")
print(f"{'kind':5s} {'Cin':>4s} {'Cout':>5s} {'taps':>4s} {'transform':>10s} {'plane':>8s} {'change':>7s}")
tot_a = tot_b = 0.0
for k in sorted(a, key=lambda k: (-k[1], k[0], k[3])):
    tot_a += a[k]; tot_b += b[k]
    print(f"{k[0]:5s} {k[1]:4d} {k[2]:5d} {k[3]:4d} {a[k]:10.3f} {b[k]:8.3f} {100 * (b[k] / a[k] - 1):+6.1f}%")
print(f"all tap-GEMMs: {tot_a:.3f} -> {tot_b:.3f} ms ({100 * (tot_b / tot_a - 1):+.1f}%)")
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for name, m in (("transform", ref), ("plane-fed", pl), ("transform", ref), ("plane-fed", pl)):
    e0.record()
    for _ in range(10):
        m(mel)
    e1.record()
    torch.cuda.synchronize()
    print(f"whole forward {name}: {e0.elapsed_time(e1) / 10:.3f} ms")

"""A/B of HiFi-GAN's narrow fused ResBlock pairs (C <= 64, not time-grouped): the persistent tile pipeline
(tcpair_narrow_kernel, the default) against two CTAs per SM (tcpair2_kernel, AGPT_NARROW_PIPE=0).
usage: narrow_pair_ab.py [B] [T] [rounds]
Creates both V1 engines in one process, alternates profiled forwards (the library's per-launch CUDA events, as
scripts/layer_profile.py reads them) and prints each pair's and each stage's minimum time over the rounds."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from audiogpt_b200 import _lib, specs
from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
T = int(sys.argv[2]) if len(sys.argv) > 2 else 800
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 5
L = _lib.lib()
h = specs.HIFIGAN_V1
sd = specs.synth_hifigan(h, 1234)
x = specs.synth_tensor((B, 80, T), seed=0, scale=2.0, shift=-4.0).cuda()


def engine(narrow):
    if narrow:
        os.environ.pop("AGPT_NARROW_PIPE", None)
    else:
        os.environ["AGPT_NARROW_PIPE"] = "0"
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    for _ in range(2):
        m(x)   # the handle reads the switch when it is created; then warm-up
    return m


engines = {"tcpair2": engine(False), "pipeline": engine(True)}
os.environ.pop("AGPT_NARROW_PIPE", None)
torch.cuda.synchronize()
best = {name: {} for name in engines}
for _ in range(rounds):
    for name, m in engines.items():
        _lib.check(L.agpt_profile_enable(1))
        m(x)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 20)
        L.agpt_profile_dump(buf, 1 << 20)
        npipe = L.agpt_profile_narrow_pipe_launches()
        _lib.check(L.agpt_profile_enable(0))
        # fields: variant G L Cin Cout ntaps span epi Wreal ms flops; a pair has epi >= 16 and both convs' taps / spans
        pairs = [f for f in (line.split() for line in buf.value.decode().splitlines())
                 if int(f[7]) >= 16 and int(f[3]) <= 64]
        for i, f in enumerate(pairs):
            k = int(f[5]) // 2
            d = int(f[6]) // (k - 1) - 1
            key = (i, int(f[3]), k, d)
            best[name][key] = min(best[name].get(key, float("inf")), float(f[9]))
        best[name]["launches"] = npipe

print(f"{torch.cuda.get_device_name()}: HiFi-GAN V1, {B} x {T} mel frames, minimum of {rounds} profiled forwards (ms)")
print(f"pipeline launches per forward: tcpair2 engine {best['tcpair2'].pop('launches')}, "
      f"pipeline engine {best['pipeline'].pop('launches')}")
print(f"{'#':>3} {'C':>3} {'k':>3} {'d':>3} {'tcpair2':>9} {'pipeline':>9} {'change':>8}")
stage = {}
for key in sorted(best["tcpair2"]):
    a, b = best["tcpair2"][key], best["pipeline"][key]
    s = stage.setdefault(key[1], [0.0, 0.0])
    s[0] += a
    s[1] += b
    print(f"{key[0]:3d} {key[1]:3d} {key[2]:3d} {key[3]:3d} {a:9.3f} {b:9.3f} {100 * (b / a - 1):+7.1f}%")
for c, (a, b) in sorted(stage.items(), reverse=True):
    print(f"stage C = {c}: {a:.3f} -> {b:.3f} ms ({100 * (b / a - 1):+.1f}%)")
ta = sum(v[0] for v in stage.values())
tb = sum(v[1] for v in stage.values())
print(f"all {len(best['tcpair2'])} pairs: {ta:.3f} -> {tb:.3f} ms ({100 * (tb / ta - 1):+.1f}%)")

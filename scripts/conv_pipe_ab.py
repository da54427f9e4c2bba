"""A/B of HiFi-GAN's plane-fed single convs and upsamplers: the persistent tile pipeline (tcconv_pipe_pl_kernel, the
default) against one tile per CTA (tcconv5_pl_kernel<128, 128>, AGPT_CONV_PIPE=0).
usage: conv_pipe_ab.py [B] [T] [rounds]
Creates both V1 engines in one process, alternates profiled forwards (the library's per-launch CUDA events, as
scripts/layer_profile.py reads them) and prints each launch's minimum time over the rounds, the C = 256 convs summed
by (k, d), and the upsamplers."""
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


def engine(pipe):
    if pipe:
        os.environ.pop("AGPT_CONV_PIPE", None)
    else:
        os.environ["AGPT_CONV_PIPE"] = "0"
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    for _ in range(2):
        m(x)   # the handle reads the switch when it is created; then warm-up
    return m


engines = {"one-tile": engine(False), "pipeline": engine(True)}
os.environ.pop("AGPT_CONV_PIPE", None)
torch.cuda.synchronize()
best = {name: {} for name in engines}
for _ in range(rounds):
    for name, m in engines.items():
        _lib.check(L.agpt_profile_enable(1))
        m(x)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 20)
        L.agpt_profile_dump(buf, 1 << 20)
        npipe = L.agpt_profile_conv_pipe_launches()
        _lib.check(L.agpt_profile_enable(0))
        # fields: variant G L Cin Cout ntaps span epi Wreal ms flops; the plane-fed single convs read > 128 channels
        convs = [f for f in (line.split() for line in buf.value.decode().splitlines())
                 if int(f[7]) < 16 and int(f[3]) > 128]
        for i, f in enumerate(convs):
            cin, cout, k, span = int(f[3]), int(f[4]), int(f[5]), int(f[6])
            kind = f"ups {cin}->{cout}" if cout != cin else f"k={k} d={span // (k - 1)}"
            key = (i, kind, int(f[7]))
            best[name][key] = min(best[name].get(key, float("inf")), float(f[9]))
        best[name]["launches"] = npipe

card = torch.cuda.get_device_name()
print(f"{card}: HiFi-GAN V1, {B} x {T} mel frames, minimum of {rounds} profiled forwards (ms)")
print(f"pipeline launches per forward: one-tile engine {best['one-tile'].pop('launches')}, "
      f"pipeline engine {best['pipeline'].pop('launches')}")
print(f"{'#':>3} {'launch':>16} {'epi':>3} {'one-tile':>9} {'pipeline':>9} {'change':>8}")
group = {}
for key in sorted(best["one-tile"]):
    a, b = best["one-tile"][key], best["pipeline"][key]
    g = group.setdefault(key[1], [0, 0.0, 0.0])
    g[0] += 1
    g[1] += a
    g[2] += b
    print(f"{key[0]:3d} {key[1]:>16} {key[2]:3d} {a:9.3f} {b:9.3f} {100 * (b / a - 1):+7.1f}%")
print("by class (sum over its launches):")
for kind, (n, a, b) in sorted(group.items()):
    print(f"  {kind:>16} x{n:<2d} {a:8.3f} -> {b:8.3f} ms ({100 * (b / a - 1):+.1f}%)")
sa = sum(v[1] for k, v in group.items() if not k.startswith("ups"))
sb = sum(v[2] for k, v in group.items() if not k.startswith("ups"))
print(f"C = 256 stage convs: {sa:.3f} -> {sb:.3f} ms ({100 * (sb / sa - 1):+.1f}%)")
ta = sum(v[1] for v in group.values())
tb = sum(v[2] for v in group.values())
print(f"all {sum(v[0] for v in group.values())} launches: {ta:.3f} -> {tb:.3f} ms ({100 * (tb / ta - 1):+.1f}%)")

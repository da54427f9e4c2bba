"""A/B of HiFi-GAN's 128-channel fused ResBlock pairs on the two-tile pipeline (tcpair_pipe_kernel): input and residual
staged by TMA with separate transform and epilogue warpgroups (the default) against one data warpgroup loading them
per thread (AGPT_PAIR_PIPE_STAGE=0).
usage: pair_pipe_ab.py [B] [T] [rounds]
Creates both V1 engines in one process, alternates profiled forwards (the library's per-launch CUDA events, as
scripts/layer_profile.py reads them) and prints each pair's and the stage's minimum time over the rounds.  Pairs are
listed in launch order: the C = 128 stage's nine (k = 3 / 7 / 11 at d = 1 / 3 / 5; k = 11, d = 5 runs
tcpair_kernel<128, 128> in both engines), then the time-grouped 128-channel views of the narrow stages (C = 64 x 2,
k = 11; C = 32 x 4, k = 7; C = 32 x 4, k = 11), whose taps and spans are counted in grouped rows."""
import ctypes as C, os, subprocess, sys
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


def engine(staged):
    if staged:
        os.environ.pop("AGPT_PAIR_PIPE_STAGE", None)
    else:
        os.environ["AGPT_PAIR_PIPE_STAGE"] = "0"
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    m = m.eval().cuda()
    for _ in range(2):
        m(x)   # the handle reads the switch when it is created; then warm-up
    return m


engines = {"per-thread": engine(False), "staged": engine(True)}
os.environ.pop("AGPT_PAIR_PIPE_STAGE", None)
torch.cuda.synchronize()
best = {name: {} for name in engines}
for _ in range(rounds):
    for name, m in engines.items():
        _lib.check(L.agpt_profile_enable(1))
        m(x)
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 20)
        L.agpt_profile_dump(buf, 1 << 20)
        npipe = L.agpt_profile_pipe_launches()
        _lib.check(L.agpt_profile_enable(0))
        # fields: variant G L Cin Cout ntaps span epi Wreal ms flops; a pair has epi >= 16 and both convs' taps / spans
        pairs = [f for f in (line.split() for line in buf.value.decode().splitlines())
                 if int(f[7]) >= 16 and int(f[3]) == 128]
        for i, f in enumerate(pairs):
            key = (i, int(f[5]), int(f[6]))   # both convs' taps and spans
            best[name][key] = min(best[name].get(key, float("inf")), float(f[9]))
        best[name]["launches"] = npipe

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
except OSError:
    card = torch.cuda.get_device_name()
print(f"{card}: HiFi-GAN V1, {B} x {T} mel frames, minimum of {rounds} profiled forwards (ms)")
print(f"pipeline launches per forward: per-thread engine {best['per-thread'].pop('launches')}, "
      f"staged engine {best['staged'].pop('launches')}")
print(f"{'#':>3} {'taps':>5} {'span':>5} {'per-thread':>10} {'staged':>9} {'change':>8}")
ta = tb = 0.0
for key in sorted(best["per-thread"]):
    a, b = best["per-thread"][key], best["staged"][key]
    ta += a
    tb += b
    print(f"{key[0]:3d} {key[1]:5d} {key[2]:5d} {a:10.3f} {b:9.3f} {100 * (b / a - 1):+7.1f}%")
print(f"all {len(best['per-thread'])} 128-channel pairs: {ta:.3f} -> {tb:.3f} ms ({100 * (tb / ta - 1):+.1f}%)")

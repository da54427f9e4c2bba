"""Dev probe: per-layer time table (CUDA events around every tapconv launch) for one model forward.
usage: layer_profile.py hifigan|diffnet|unet [B] [T] [--each]
--each also lists every launch in issue order (a fused ResBlock pair is one line: epi >= 16, taps and spans of both
convs summed), so pairs that share a shape but not a dilation can be told apart."""
import ctypes as C, os, sys, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from audiogpt_b200 import _lib, specs
L = _lib.lib()
each = "--each" in sys.argv
argv = [a for a in sys.argv if a != "--each"]
which = argv[1] if len(argv) > 1 else "hifigan"
B = int(argv[2]) if len(argv) > 2 else 8
if which == "hifigan":
    from audiogpt_b200.modules.hifigan.hifigan import HifiGanGenerator
    h = specs.HIFIGAN_V1
    m = HifiGanGenerator(h); m.load_state_dict(specs.synth_hifigan(h, 1234)); m = m.eval().cuda()
    T = int(argv[3]) if len(argv) > 3 else 400
    x = specs.synth_tensor((B, 80, T), seed=0, scale=2.0, shift=-4.0).cuda()
    run = lambda: m(x)
elif which == "diffnet":
    from audiogpt_b200.modules.diff.net import DiffNet
    h = specs.DIFFNET_BASE
    m = DiffNet(h); m.load_state_dict(specs.synth_diffnet(h, 1)); m = m.eval().cuda()
    spec = torch.randn(B, 1, 80, 400).cuda(); cond = torch.randn(B, 256, 400).cuda(); t = torch.full((B,), 50).cuda()
    run = lambda: m(spec, t, cond)
else:
    from audiogpt_b200.ldm.modules.diffusionmodules.openaimodel import UNetModel
    h = specs.UNET_TXT2AUDIO
    m = UNetModel(**h) if isinstance(h, dict) else UNetModel(h)
    m.load_state_dict(specs.synth_unet(h, 1)); m = m.eval().cuda()
    x = torch.randn(B, 4, 10, 78).cuda(); ctx = torch.randn(B, 77, 1024).cuda(); t = torch.full((B,), 500).cuda()
    run = lambda: m(x, t, context=ctx)
for _ in range(2): run()
torch.cuda.synchronize()
_lib.check(L.agpt_profile_enable(1))
run()
buf = C.create_string_buffer(1 << 20)
n = L.agpt_profile_dump(buf, 1 << 20)
conv_pipe = L.agpt_profile_conv_pipe_launches()
_lib.check(L.agpt_profile_enable(0))
agg = collections.OrderedDict()
tot = 0.0
lines = buf.value.decode().splitlines()
for line in lines:
    v, G, Ln, Cin, Cout, nt, span, epi, Wr, ms, fl = line.split()
    key = (int(G), int(Ln), int(Cin), int(Cout), int(nt), int(epi), int(Wr))
    a = agg.setdefault(key, [0, 0.0, 0.0]); a[0] += 1; a[1] += float(ms); a[2] += float(fl); tot += float(ms)
print(f"{which} B={B}: {tot:.3f} ms in {sum(a[0] for a in agg.values())} tapconv launches, "
      f"{conv_pipe} of them plane-fed convs on the tile pipeline")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"  G={k[0]:3d} L={k[1]:7d} Cin={k[2]:5d} Cout={k[3]:5d} taps={k[4]:2d} epi={k[5]:2d} W={k[6]:3d}  n={a[0]:3d}  {a[1]*1e3:9.1f} us  {a[1]/tot*100:5.1f}%  {a[2]/a[1]/1e9:7.1f} TF")
if each:
    print("every launch in issue order:")
    for i, line in enumerate(lines):
        v, G, Ln, Cin, Cout, nt, span, epi, Wr, ms, fl = line.split()
        kind = "pair" if int(epi) >= 16 else "conv"
        print(f"  #{i:3d} {kind} G={int(G):3d} L={int(Ln):7d} Cin={int(Cin):5d} Cout={int(Cout):5d} taps={int(nt):2d} "
              f"span={int(span):3d} epi={int(epi):2d}  {float(ms)*1e3:9.1f} us")

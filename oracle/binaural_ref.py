"""Functional restatement of the Binaural tool's network (mono2binaural/src/models.py BinauralNetwork -> Warpnet, eval
mode) and of the tool's chunk loop (audio-chatgpt.py:729-766), in plain torch.

The reference rotates the mouth offset with scipy on the host; here the quaternion step is fp64 torch (normalise, build
the rotation matrix, apply its transpose), rounded to fp32 as ``th.Tensor(...)`` does, so no scipy is needed.
``dtype=torch.float64`` runs every step in fp64 (the GPU tests' accuracy yardstick); the default fp32 follows the
reference's own op order.  ``host_rotation=True`` moves the quaternions to the host for the rotation and back, as the
reference does (one device synchronisation per call)."""
import torch
import torch.nn.functional as F

MOUTH = (0.09, 0.0, -0.20)
EARS = ((0.0, -0.08, -0.22), (0.0, 0.08, -0.22))
SPEED_OF_SOUND = 343.0
SR = 48000


def mouth(view, dtype=torch.float32, host_rotation=False):
    """view [B, 7, K] -> the mouth offset rotated by the inverse of each frame's quaternion, [B, 3, K] in ``dtype``."""
    q = view[:, 3:7, :].transpose(1, 2).reshape(-1, 4)
    if host_rotation:
        q = q.cpu()
    zero = (q == 0).all(dim=1, keepdim=True)
    q = (q + zero.to(q.dtype)).double()
    q = q / q.pow(2).sum(dim=1, keepdim=True).sqrt()
    x, y, z, w = q.unbind(1)
    m = torch.stack([
        torch.stack([x * x - y * y - z * z + w * w, 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
        torch.stack([2 * (x * y + z * w), -x * x + y * y - z * z + w * w, 2 * (y * z - x * w)], -1),
        torch.stack([2 * (x * z - y * w), 2 * (y * z + x * w), -x * x - y * y + z * z + w * w], -1)], -2)
    off = torch.tensor(MOUTH, dtype=torch.float64, device=m.device)
    r = torch.einsum("nji,j->ni", m, off).to(dtype)
    B, _, K = view.shape
    return r.reshape(B, K, 3).transpose(1, 2).contiguous().to(view.device)


def geometric(view, dtype=torch.float32, host_rotation=False):
    """[B, 2, K]: (-distance / 343) * 48000 per ear at frame rate."""
    v = view.to(dtype)
    p = v[:, 0:3, :] + mouth(view, dtype, host_rotation)
    ds = [p - torch.tensor(e, dtype=dtype, device=v.device)[None, :, None] for e in EARS]
    d = torch.stack(ds, dim=1)                    # [B, 2, 3, K]
    dist = torch.sum(d ** 2, dim=2) ** 0.5
    return -dist / SPEED_OF_SOUND * SR


def neural(sd, cfg, view, dtype=torch.float32):
    """[B, 2, K]: the warpnet's causal convs and its 1 x 1 head at frame rate."""
    h = view.to(dtype)
    for l in range(int(cfg["layers"])):
        h = F.relu(F.conv1d(F.pad(h, [1, 0]), sd[f"warper.layers.{l}.weight"].to(h), sd[f"warper.layers.{l}.bias"].to(h)))
    return F.conv1d(h, sd["warper.linear.weight"].to(h), sd["warper.linear.bias"].to(h))


def frame_field(sd, cfg, view, dtype=torch.float32, host_rotation=False):
    """[B, 2, K]: geometric + neural warp per frame.  Nearest interpolation picks the same frame for both parts, so this
    selected per sample is the reference's per-sample warpfield."""
    return geometric(view, dtype, host_rotation) + neural(sd, cfg, view, dtype)


def warp(mono, field):
    """mono [B, 1, T], frame field [B, 2, K] -> [B, 2, T]: nearest selection, -relu(-w), + arange, clamp, cummax, lerp.
    The frame field may be fp64; the selection is always the reference's fp32 rule."""
    T = mono.shape[-1]
    if field.shape[-1] == 0:
        raise ValueError("empty view: F.interpolate needs at least one frame")
    # the frame each sample selects, by the rule the reference's fp32 F.interpolate follows (an fp64 input would take
    # its scale in fp64 and pick other frames at a few boundaries of a long row)
    sel = F.interpolate(torch.arange(field.shape[-1], dtype=torch.float32, device=field.device)[None, None], size=T)[0, 0].long()
    w = field[..., sel]
    w = -F.relu(-w)
    pos = torch.clamp(w + torch.arange(T, dtype=w.dtype, device=w.device)[None, None, :], min=0, max=T - 1)
    pos = torch.cummax(pos, dim=-1)[0]
    x = torch.cat([mono, mono], dim=1).to(w.dtype)
    lo = pos.floor().long()
    hi = torch.clamp(pos.ceil().long(), max=T - 1)
    a = pos - pos.floor()
    return (1 - a) * torch.gather(x, 2, lo) + a * torch.gather(x, 2, hi)


def forward(sd, cfg, mono, view, dtype=torch.float32, host_rotation=False):
    """BinauralNetwork.forward: mono [B, 1, T], view [B, 7, K] -> [B, 2, T]."""
    return warp(mono, frame_field(sd, cfg, view, dtype, host_rotation))


def tool(mono, view, net, chunk_size=48000, rec_field=800):
    """The Binaural tool's inference body after loading: mono [1, L], view [7, Kv] -> the clamped [2, L'] it saves.
    ``net(mono [1, 1, T], view [1, 7, K]) -> [1, 2, T]`` is the network (this module's forward or a drop-in)."""
    if not view.shape[-1] * 400 == mono.shape[-1]:
        mono = mono[:, :(mono.shape[-1] // 400) * 400]
        if view.shape[1] * 400 > mono.shape[1]:
            m_a = view.shape[1] - mono.shape[-1] // 400
            view = view[:, m_a:m_a + (mono.shape[-1] // 400)]
    chunks = [{"mono": mono[:, max(0, i - rec_field):i + chunk_size],
               "view": view[:, max(0, i - rec_field) // 400:(i + chunk_size) // 400]}
              for i in range(0, mono.shape[-1], chunk_size)]
    outs = []
    for i, ch in enumerate(chunks):
        with torch.no_grad():
            m = ch["mono"].unsqueeze(0)
            b = net(m, ch["view"].unsqueeze(0)).squeeze(0)
            if i > 0:
                b = b[:, -(m.shape[-1] - rec_field):]
        outs.append(b)
    return torch.clamp(torch.cat(outs, dim=-1), min=-1, max=1)

"""Attention diagnostics (called from tools/gpu_diag.py)."""
import torch

from dalle_mtf_b200 import ops

DEV = "cuda"


def ref_attn(qkv, scale):
    # qkv: [B,S,3,H,dh] float (requires_grad)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]              # [B,S,H,dh]
    s = torch.einsum("bihe,bjhe->bhij", q, k) * scale
    S = q.shape[1]
    mask = torch.triu(torch.ones(S, S, dtype=torch.bool), 1)
    s = s.masked_fill(mask, float("-inf"))
    lse = torch.logsumexp(s, -1)                                     # [B,H,S]
    p = torch.softmax(s, -1)
    o = torch.einsum("bhij,bjhe->bihe", p, v)
    return o, lse


def run(report, guarded):
    @guarded
    def case(B, S, H, dh, scale, mag, seed, perf=False):
        g = torch.Generator().manual_seed(seed)
        qkv = (torch.randn(B, S, 3, H, dh, generator=g) * mag).to(torch.bfloat16)
        dout = (torch.randn(B, S, H, dh, generator=g)).to(torch.bfloat16)
        qf = qkv.float().requires_grad_(True)
        o_ref, lse_ref = ref_attn(qf, scale)
        o_ref.backward(dout.float())
        qd, dd = qkv.to(DEV), dout.to(DEV)
        out = torch.zeros(B, S, H, dh, dtype=torch.bfloat16, device=DEV)
        lse = torch.zeros(B, H, S, device=DEV)
        ops.attn_fwd(qd, out, lse, B, S, H, dh, scale)
        torch.cuda.synchronize()
        tag = f"attn B={B} S={S} H={H} dh={dh} scale={scale}"
        report(tag + " fwd out", out.reshape(B * S, H * dh), o_ref.reshape(B * S, H * dh), 1e-2)
        report(tag + " fwd lse", lse.reshape(B * H, S), lse_ref.reshape(B * H, S), 1e-3)
        dqkv = torch.zeros_like(qd)
        delta = torch.zeros(B, H, S, device=DEV)
        dq_acc = torch.zeros(1, device=DEV)
        ops.attn_bwd(qd, out, dd, lse, dq_acc, delta, dqkv, B, S, H, dh, scale)
        torch.cuda.synchronize()
        gref = qf.grad
        for i, nm in enumerate("qkv"):
            report(tag + f" bwd d{nm}", dqkv[:, :, i].reshape(B * S, H * dh), gref[:, :, i].reshape(B * S, H * dh),
                   2e-2)

    case(1, 128, 1, 128, 1.0, 0.3, 0)
    case(1, 128, 1, 64, 1.0, 0.4, 1)
    case(2, 256, 2, 128, 1.0, 0.3, 2)
    case(1, 300, 3, 64, 0.125, 1.0, 3)
    case(1, 333, 2, 128, 0.0884, 1.0, 4)
    case(2, 1280, 4, 128, 1.0, 0.25, 5)
    case(1, 640, 2, 128, 1.0, 1.2, 6)      # peaked softmax: the running maximum moves by > 2^8 (lazy rescale path)
    case(1, 520, 3, 64, 1.0, 1.5, 7)
    case(1, 129, 1, 128, 1.0, 0.5, 8)      # second tile has a single valid row
    case(2, 1280, 3, 64, 0.125, 1.0, 9)
    # more (tile, head, batch) blocks than SMs
    case(8, 1280, 5, 128, 1.0, 0.25, 10)
    case(6, 1280, 8, 64, 0.125, 1.0, 11)
    case(5, 640, 8, 128, 1.0, 1.2, 12)

    @guarded
    def perf(B, S, H, dh):
        qkv = (torch.randn(B, S, 3, H, dh, device=DEV) * 0.3).to(torch.bfloat16)
        dout = torch.randn(B, S, H, dh, device=DEV).to(torch.bfloat16)
        out = torch.zeros(B, S, H, dh, dtype=torch.bfloat16, device=DEV)
        lse = torch.zeros(B, H, S, device=DEV)
        dqkv = torch.zeros_like(qkv)
        delta = torch.zeros(B, H, S, device=DEV)
        dq_acc = torch.zeros(1, device=DEV)
        fl = 4.0 * S * S * dh * B * H / 2
        for name, fn, mult in (("fwd", lambda: ops.attn_fwd(qkv, out, lse, B, S, H, dh, 1.0), 1.0),
                               ("bwd", lambda: ops.attn_bwd(qkv, out, dout, lse, dq_acc, delta, dqkv, B, S, H, dh, 1.0),
                                2.5)):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            print(f"[PERF] attn {name} B={B} S={S} H={H} dh={dh}: {ms:.3f} ms  {fl * mult / ms / 1e9:.1f} TFLOP/s (causal-algorithmic)",
                  flush=True)

    perf(32, 1280, 4, 128)
    perf(16, 1280, 16, 64)

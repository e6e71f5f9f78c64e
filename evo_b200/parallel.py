"""Sequence-parallel StripedHyena forward for contexts that do not fit / are too slow on one
GPU (BASELINE.json configs[2]: evo-1-131k-base, batch 1 x 131072 nt over 8 GPUs).

The reference has no multi-GPU code at all (SURVEY.md section 5); this is new.  One process per
GPU, weights replicated, every rank holds a contiguous slice of the sequence.  Token-local
work (embedding, RMSNorm, every GEMM, the gated MLP, unembed) needs no communication.

  Hyena layer      halo: the two z rows preceding the shard (all-gather of 2 rows per rank);
                   carry: each rank scans its shard from a zero state and emits the end state
                   (B, D, 8) complex64 -> ONE all-gather of 256 KB*B per rank -> every rank folds
                   S_in = sum_{q<r} p^{(r-1-q) Lr} E_q (evo_hyena_combine_states) and runs the
                   output scan from S_in.  Exact: it is the modal recurrence itself.
  Attention layer  head <-> sequence re-shard (Ulysses): one all-to-all turns the local
                   (Lr tokens x H heads) qkv into (L tokens x H/P heads), every rank runs the
                   full-length causal kernel for its heads (perfectly balanced: a K/V all-gather
                   would leave the last rank with 1.9x the average causal work), a second
                   all-to-all returns the context to sequence-sharded layout.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch
import torch.distributed as dist

from . import _lib
from ._lib import EPI_BIAS, EPI_BIAS_RESID, EPI_BIAS_ROPE, AttnParams, HyenaParams, check, ptr
from .stripedhyena.model import ATTN_VARIANT


# attention re-shard through our own NVLink peer stores (PeerUlysses) instead of NCCL all-to-alls; "0" = NCCL Ulysses.
PEER_ULYSSES = os.environ.get("EVO_B200_PEER_ULYSSES", "1") != "0"


def _all_gather(t: torch.Tensor, world: int, group=None) -> torch.Tensor:
    out = torch.empty((world,) + tuple(t.shape), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous(), group=group)
    return out


class PeerCarry:
    """Symmetric (peer-mapped) buffers for the Hyena halo / end-state exchange: a ring of NBUF slot sets,
    each [ends: world x end_bytes | halo: halo_bytes | end_flags: world x i32 | halo_flags: world x i32].
    Ranks push with evo_peer_publish (NVLink stores + release flag) and consume after evo_peer_wait."""
    NBUF = 8

    def __init__(self, world, rank, B, d, S, dev, group):
        import torch.distributed._symmetric_memory as symm
        self.world, self.rank = world, rank
        self.end_bytes = B * d * S * 2 * 4
        self.halo_bytes = B * 2 * 3 * d * 2
        al = lambda n: (n + 255) // 256 * 256
        self.off_halo = al(world * self.end_bytes)
        self.off_eflag = self.off_halo + al(self.halo_bytes)
        self.off_hflag = self.off_eflag + al(world * 4)
        self.set_bytes = self.off_hflag + al(world * 4)
        self.buf = symm.empty(self.NBUF * self.set_bytes, dtype=torch.uint8, device=dev)
        self.buf.zero_()
        torch.cuda.synchronize(dev)
        self.hdl = symm.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        mk = lambda vals: torch.tensor(vals, dtype=torch.int64, device=dev)
        self.ends_dsts = [mk([p + k * self.set_bytes for p in ptrs]) for k in range(self.NBUF)]
        self.halo_dsts = [mk([p + k * self.set_bytes + self.off_halo for p in ptrs]) for k in range(self.NBUF)]
        self.eflag_dsts = [mk([p + k * self.set_bytes + self.off_eflag for p in ptrs]) for k in range(self.NBUF)]
        self.hflag_dsts = [mk([p + k * self.set_bytes + self.off_hflag for p in ptrs]) for k in range(self.NBUF)]
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.epoch = 0
        self.key = (world, rank, B, d, S, str(dev))

    def local(self, k, off, nbytes):
        return self.buf[k * self.set_bytes + off: k * self.set_bytes + off + nbytes]


class PeerUlysses:
    """Symmetric (peer-mapped) buffers for the attention layers' head<->sequence re-shard WITHOUT NCCL and without permute
    copies (B == 1): the Wqkv GEMM's epilogue stores every (q|k|v, head) tile straight into the owning rank's `full`
    buffer over NVLink (evo_gemm peer-scattered output, rotary applied on the way), the attention kernel's epilogue stores
    every query row straight into the token-owning rank's `ctx` buffer; two flag rounds (evo_peer_publish with no payload /
    evo_peer_wait) tell a rank when all of its inputs have landed.  `full` is double-buffered: a rank may enter the next
    attention layer while a slower peer still reads the previous one (it cannot get two layers ahead: the layer in between
    needs that peer's q/k/v).  Layout per rank: [full0 | full1 | ctx | q-flags | c-flags]."""

    def __init__(self, world, rank, Lr, d, H, dev, group):
        import torch.distributed._symmetric_memory as symm
        hd = d // H
        self.world, self.rank, self.Lr, self.d = world, rank, Lr, d
        self.Hl, self.dl = H // world, (H // world) * hd
        self.L = Lr * world
        al = lambda n: (n + 255) // 256 * 256
        self.full_bytes = al(self.L * 3 * self.dl * 2)
        self.ctx_bytes = al(Lr * d * 2)
        self.off_ctx = 2 * self.full_bytes
        self.off_qflag = self.off_ctx + self.ctx_bytes
        self.off_cflag = self.off_qflag + al(world * 4)
        total = self.off_cflag + al(world * 4)
        self.buf = symm.empty(total, dtype=torch.uint8, device=dev)
        self.buf[self.off_qflag:].zero_()
        torch.cuda.synchronize(dev)
        self.hdl = symm.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        ptrs = [int(x) for x in self.hdl.buffer_ptrs]
        arr = lambda vals: (C.c_void_p * world)(*vals)
        self.full_ptrs = [arr([x + k * self.full_bytes for x in ptrs]) for k in range(2)]
        self.ctx_ptrs = arr([x + self.off_ctx for x in ptrs])
        mk = lambda vals: torch.tensor(vals, dtype=torch.int64, device=dev)
        self.dummy_dsts = mk(ptrs)                                            # payload-free publish: nothing is copied
        self.qflag_dsts = mk([x + self.off_qflag for x in ptrs])
        self.cflag_dsts = mk([x + self.off_cflag for x in ptrs])
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.epoch = 0
        self.calls = 0
        self.key = (world, rank, Lr, d, H, str(dev))

    def full(self, k):
        return self.buf[k * self.full_bytes: k * self.full_bytes + self.L * 3 * self.dl * 2].view(torch.bfloat16)

    def ctx(self):
        return self.buf[self.off_ctx: self.off_ctx + self.Lr * self.d * 2].view(torch.bfloat16).view(self.Lr, self.d)

    def signal_and_wait(self, model, lib, which, stream):
        """All ranks: 'my stores of this phase are done' -> every peer; then wait until every rank has said so."""
        dsts = self.qflag_dsts if which == "q" else self.cflag_dsts
        off = self.off_qflag if which == "q" else self.off_cflag
        w = self.world
        model._record("comm/peer_flags", 0.0, lambda: (
            check(lib.evo_peer_publish(ptr(self.counter), 0, ptr(self.dummy_dsts), ptr(dsts), 0, self.rank, 0, w - 1, self.epoch, ptr(self.counter), stream()), "evo_peer_publish(flags)"),
            check(lib.evo_peer_wait(ptr(self.buf[off: off + w * 4]), 0, w - 1, self.epoch, stream()), "evo_peer_wait(flags)")))


def _peer_attention(model, lib, pu, i, xn, mha, u, B, Lr, H, hd, rank, world, stream):
    """One sequence-parallel attention layer with the re-shard fused into the GEMM / attention epilogues (PeerUlysses).
    xn (Lr, D) = pre-norm output of block i; returns ctx (Lr, D), this rank's tokens x all heads, ready for out_proj."""
    d = H * hd
    k = pu.calls % 2
    pu.calls += 1
    pu.epoch += 1
    cos_p, sin_p = model._rope_at(rank * Lr, Lr, xn.device)
    # Wqkv: bias + rotary + scatter to the head-owning ranks, tile by tile while the GEMM runs
    model._gemm(xn, model.linear_weight(i, "in"), None, Lr, 3 * d, d, EPI_BIAS_ROPE, bias=mha.Wqkv.bias, ldc=3 * pu.dl, rope=(cos_p, sin_p, Lr, 2 * d),
                peers=(pu.full_ptrs[k], world, d, pu.dl, rank * Lr))
    pu.signal_and_wait(model, lib, "q", stream)
    full = pu.full(k)                                   # (L, 3, Hl, hd): my heads, the whole sequence
    L, dl = pu.L, pu.dl
    ap = AttnParams(out=None, B=1, Lq=L, Lk=L, H=pu.Hl, hd=hd, q_pos0=0, softmax_scale=1.0 / math.sqrt(hd))
    ap.q, ap.q_tok_stride, ap.q_batch_stride = full.data_ptr(), 3 * dl, L * 3 * dl
    ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride = full.data_ptr() + dl * 2, full.data_ptr() + 2 * dl * 2, 3 * dl, L * 3 * dl
    ap.out_peers, ap.n_out_peers, ap.out_rows_per_peer, ap.out_row_stride, ap.out_col0 = C.cast(pu.ctx_ptrs, C.c_void_p), world, Lr, d, rank * dl
    causal_flops = 4.0 * pu.Hl * hd * (L * (L + 1) / 2.0)
    model._record("attn", causal_flops, lambda: check(lib.evo_attn_fwd_ws(C.byref(ap), ATTN_VARIANT, None, 0, stream()), "evo_attn_fwd(peer)"))
    pu.signal_and_wait(model, lib, "c", stream)
    return pu.ctx()


def _ulysses_attention(model, lib, qkv, ctx, B, Lr, H, hd, rank, world, group, stream):
    """qkv (B*Lr, 3*H*hd) rotary-applied, sequence-sharded -> ctx (B*Lr, H*hd), sequence-sharded."""
    if H % world != 0:
        raise _lib.EvoError(f"sequence-parallel attention needs heads ({H}) divisible by the world size ({world})")
    Hl = H // world
    dev = qkv.device
    L = Lr * world
    # (B, Lr, 3, P, Hl, hd) -> (P, B, Lr, 3, Hl, hd): chunk p goes to rank p
    box = {}
    model._record("comm/permute", 2.0 * qkv.numel() * 2, lambda: box.__setitem__("send", qkv.view(B, Lr, 3, world, Hl, hd).permute(3, 0, 1, 2, 4, 5).contiguous()))
    send = box["send"]
    recv = torch.empty_like(send)                     # (P = source rank = sequence chunk, B, Lr, 3, Hl, hd)
    model._record("comm/all_to_all", send.numel() * 2.0 * (world - 1) / world, lambda: dist.all_to_all_single(recv, send, group=group))
    if B == 1:
        full = recv.view(1, L, 3, Hl, hd)             # source-rank order is sequence order
    else:
        model._record("comm/permute", 2.0 * recv.numel() * 2, lambda: box.__setitem__("full", recv.permute(1, 0, 2, 3, 4, 5).reshape(B, L, 3, Hl, hd).contiguous()))
        full = box["full"]
    dl = Hl * hd
    out = torch.empty(B, L, dl, dtype=torch.bfloat16, device=dev)
    ap = AttnParams(out=out.data_ptr(), B=B, Lq=L, Lk=L, H=Hl, hd=hd, q_pos0=0, softmax_scale=1.0 / math.sqrt(hd))
    ap.q, ap.q_tok_stride, ap.q_batch_stride = full.data_ptr(), 3 * dl, L * 3 * dl
    ap.k, ap.v, ap.kv_tok_stride, ap.kv_batch_stride = full.data_ptr() + dl * 2, full.data_ptr() + 2 * dl * 2, 3 * dl, L * 3 * dl
    causal_flops = 4.0 * B * Hl * hd * (L * (L + 1) / 2.0)
    model._launch_ws("attn", causal_flops, "evo_attn_fwd", lib.evo_attn_fwd_workspace, lib.evo_attn_fwd_ws, ap, ATTN_VARIANT)
    # back: (B, P, Lr, Hl*hd) -> chunk p (its tokens, my heads) to rank p
    if B == 1:
        send2 = out.view(world, B, Lr, dl)            # chunk p = tokens of rank p: already contiguous
    else:
        model._record("comm/permute", 2.0 * out.numel() * 2, lambda: box.__setitem__("send2", out.view(B, world, Lr, dl).permute(1, 0, 2, 3).contiguous()))
        send2 = box["send2"]
    recv2 = torch.empty_like(send2)                   # (P = head group, B, Lr, dl)
    model._record("comm/all_to_all", send2.numel() * 2.0 * (world - 1) / world, lambda: dist.all_to_all_single(recv2, send2, group=group))
    model._record("comm/permute", 2.0 * recv2.numel() * 2, lambda: ctx.view(B, Lr, world, dl).copy_(recv2.permute(1, 2, 0, 3)))


def sequence_parallel_forward(model, ids_local: torch.Tensor, rank: int, world: int, group=None, transport: str = "auto"):
    """ids_local: (B, L/world) slice `rank` of the token ids.  Returns the logits of the slice,
    (B, L/world, V) bf16.  Stateless (scoring) forward only.
    transport: how the Hyena halo / end states travel: "peer" = pushed into peer-mapped symmetric memory by
    our own kernels over NVLink, "nccl" = two all-gathers per layer, "auto" = peer when available."""
    model._ensure_packed()
    cfg = model.config
    lib = _lib.lib()
    dev = ids_local.device
    B, Lr = ids_local.shape
    M = B * Lr
    d, H, V = cfg.hidden_size, cfg.num_attention_heads, cfg.vocab_size
    hd = d // H
    S = cfg.state_size
    stream = model._stream
    pc = None
    if transport in ("auto", "peer") and world > 1:
        pc = getattr(model, "_peer_carry", None)
        if pc is None or (pc is not False and pc.key != (world, rank, B, d, S, str(dev))):
            try:
                pc = PeerCarry(world, rank, B, d, S, dev, group)
            except Exception as ex:  # symmetric memory unavailable on this system
                pc = None
                model._peer_carry_error = repr(ex)
            # the transport is a collective decision: one rank on NCCL all-gathers while the others spin on peer flags would
            # hang, so every rank learns whether ALL of them have the peer path
            pu = None
            rope_fused = all(model._rope_fused(model.blocks[j].inner_mha_cls) for j in model._attn_idxs)    # the peer scatter is that epilogue's
            if PEER_ULYSSES and pc is not None and B == 1 and H % world == 0 and hd == 128 and rope_fused:
                try:
                    pu = PeerUlysses(world, rank, Lr, d, H, dev, group)
                except Exception as ex:  # noqa
                    pu = None
                    model._peer_carry_error = repr(ex)
            okv = [1 if pc is not None else 0, 1 if pu is not None else 0]
            ok2 = torch.tensor(okv, dtype=torch.int32, device=dev)
            dist.all_reduce(ok2, op=dist.ReduceOp.MIN, group=group)
            model._peer_ulysses = pu if int(ok2[1].item()) == 1 else None
            ok = ok2[:1]
            if int(ok.item()) == 0:
                if transport == "peer":
                    raise _lib.EvoError("peer-memory transport unavailable on at least one rank: " + str(getattr(model, "_peer_carry_error", "")))
                pc = None
            model._peer_carry = pc if pc is not None else False     # False = decided: NCCL (do not retry every forward)
        if pc is False:
            pc = None
        if pc is not None:
            model._record("comm/barrier", 0.0, lambda: dist.barrier(group))          # nobody is still reading ring slots of the previous forward
    since_sync = 0
    pu = getattr(model, "_peer_ulysses", None) if (pc is not None and transport in ("auto", "peer")) else None
    if pu is not None and pu.key != (world, rank, Lr, d, H, str(dev)):
        pu = None
    with torch.cuda.device(dev), torch.no_grad():
        u = model._embed(ids_local.contiguous())
        for i, blk in enumerate(model.blocks):
            xn = torch.empty_like(u)
            model._rmsnorm(u, blk.pre_norm.scale, xn, M)
            if i in model._attn_idxs and pu is not None:
                mha = blk.inner_mha_cls
                ctx = _peer_attention(model, lib, pu, i, xn, mha, u, B, Lr, H, hd, rank, world, stream)
                since_sync = 0           # the flag rounds are global synchronisation points
                u2 = model._out_proj(i, mha, ctx, u)
            elif i in model._attn_idxs:
                mha = blk.inner_mha_cls
                qkv = torch.empty(M, 3 * d, dtype=torch.bfloat16, device=dev)
                model._qkv_rope(i, xn, mha, qkv, B, Lr, model._rope_at(rank * Lr, Lr, dev))
                ctx = xn
                _ulysses_attention(model, lib, qkv, ctx, B, Lr, H, hd, rank, world, group, stream)
                since_sync = 0           # the all-to-all is a global synchronisation point
                u2 = model._out_proj(i, mha, ctx, u)
            else:
                f = blk.filter
                z = torch.empty(M, 3 * d, dtype=torch.bfloat16, device=dev)
                model._gemm(xn, model.linear_weight(i, "in"), z, M, 3 * d, d, EPI_BIAS, bias=blk.projections.bias)
                tail = z.view(B, Lr, 3 * d)[:, -2:].contiguous()
                if pc is not None:
                    if since_sync == pc.NBUF:
                        model._record("comm/barrier", 0.0, lambda: dist.barrier(group))
                        since_sync = 0
                    k = since_sync
                    since_sync += 1
                    pc.epoch += 1
                    if rank + 1 < world:
                        model._record("comm/peer_halo", float(pc.halo_bytes), lambda: check(lib.evo_peer_publish(
                            ptr(tail), pc.halo_bytes, ptr(pc.halo_dsts[k]), ptr(pc.hflag_dsts[k]), 0, rank, rank + 1, rank + 1,
                            pc.epoch, ptr(pc.counter), stream()), "evo_peer_publish(halo)"))
                    halo = None
                    if rank > 0:
                        model._record("comm/peer_halo", 0.0, lambda: check(lib.evo_peer_wait(
                            ptr(pc.local(k, pc.off_hflag, world * 4)), rank - 1, rank - 1, pc.epoch, stream()), "evo_peer_wait(halo)"))
                        halo = pc.local(k, pc.off_halo, pc.halo_bytes)
                else:
                    box = {}
                    model._record("comm/all_gather", float(tail.numel() * 2 * (world - 1)), lambda: box.__setitem__("t", _all_gather(tail, world, group)))   # (W, B, 2, 3D)
                    tails = box["t"]
                    halo = tails[rank - 1].contiguous() if rank > 0 else None
                end = torch.empty(B, d, S, 2, dtype=torch.float32, device=dev)
                hp = HyenaParams(z=z.data_ptr(), y=None, **f.ptrs(), B=B, L=Lr, D=d, S=S, nheads=H,
                                 halo=halo.data_ptr() if halo is not None else None, state_in=None, state_out=end.data_ptr(), fir_state_out=None,
                                 force_segments=0, state_only=1)
                ws, n = model._launch_ws("hyena_state", 4.0 * B * Lr * d, "evo_hyena_fwd(state)", lib.evo_hyena_fwd_workspace, lib.evo_hyena_fwd, hp)
                if pc is not None:
                    if rank + 1 < world:   # only later shards need my end state
                        model._record("comm/peer_state", float(pc.end_bytes * (world - 1 - rank)), lambda: check(lib.evo_peer_publish(
                            ptr(end), pc.end_bytes, ptr(pc.ends_dsts[k]), ptr(pc.eflag_dsts[k]), pc.end_bytes, rank, rank + 1, world - 1,
                            pc.epoch, ptr(pc.counter), stream()), "evo_peer_publish(end)"))
                    if rank > 0:
                        model._record("comm/peer_state", 0.0, lambda: check(lib.evo_peer_wait(
                            ptr(pc.local(k, pc.off_eflag, world * 4)), 0, rank - 1, pc.epoch, stream()), "evo_peer_wait(end)"))
                    ends = pc.local(k, 0, world * pc.end_bytes)
                else:
                    box = {}
                    model._record("comm/all_gather", float(end.numel() * 4 * (world - 1)), lambda: box.__setitem__("e", _all_gather(end, world, group)))   # (W, B, D, S, 2)
                    ends = box["e"]
                s_in = torch.empty_like(end)
                model._record("hyena_combine", 0.0, lambda: check(lib.evo_hyena_combine_states(ptr(ends), ptr(s_in), ptr(f.poles), rank, world, Lr, B, d, S, stream()), "evo_hyena_combine_states"))
                y = xn
                # output pass: same geometry, so the per-segment end states of the carry pass are reused from `ws`
                hp.y, hp.state_in, hp.state_out, hp.state_only, hp.reuse_segment_states = y.data_ptr(), s_in.data_ptr(), None, 0, 1
                model._record("hyena", 8.0 * B * Lr * d, lambda: check(lib.evo_hyena_fwd(C.byref(hp), ptr(ws), n, stream()), "evo_hyena_fwd"))
                u2 = torch.empty_like(u)
                model._gemm(y, model.linear_weight(i, "out"), u2, M, d, d, EPI_BIAS_RESID, bias=blk.out_filter_dense.bias, resid=u)
            u = model._mlp_residual(i, blk, u2, M)
        logits = model._logits(model._final_norm(u))
    return logits.view(B, Lr, V)

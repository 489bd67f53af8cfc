"""Sequence-parallel (DeepSpeed-Ulysses) execution of the Wan DiT on libfvb200: one process per GPU,
torch.distributed (NCCL over NVLink) for the two all-to-alls around self-attention and the final gather.

Mirrors the reference's scheme (fastvideo/distributed/communication_op.py:28-91,
fastvideo/distributed/device_communicators/base_device_communicator.py:41-193, fastvideo/attention/layer.py:82-245,
fastvideo/models/dits/wanvideo.py:693,758): tokens are sharded in contiguous chunks (zero padded to a multiple of
the group size), every self-attention swaps "my tokens, all heads" for "all tokens, my heads" and back, and the
sequence is gathered once at the end.

What is different (results identical):
  * no pack / unpack copies around the all-to-all: the QKV(+gate) GEMM writes each head straight into the send
    buffer slot of the rank that owns it ([dest][token][q|k|v|g][local head][d], fvb_linear_bf16_sp), the attention
    kernel reads the receive buffer in place through strided TMA descriptors, and the out-projection GEMM reads
    the second receive buffer as a K-segmented A operand;
  * RoPE is applied before the exchange (it is per token and per head, so it commutes with the all-to-all;
    the reference applies it after, on the full sequence: attention/layer.py:130-132);
  * the final projection runs on the local shard and only [S, 64] outputs are gathered, instead of gathering the
    [S, D] hidden states first (wanvideo.py:758-759) -- proj_out is token-wise, so this commutes too.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import torch
import torch.distributed as dist


# ----------------------------------------------------------------------------------------------------------------
# pure layout arithmetic (CPU-testable; used by the gloo tests and by the CUDA path)
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class SPPlan:
    world: int
    rank: int
    seq_len: int          # original (unpadded) number of tokens
    num_heads: int
    head_dim: int
    n_proj: int           # 3 (q,k,v) or 4 (q,k,v,gate)

    @property
    def local_seq(self) -> int:  # communication_op.py:77-89: pad to a multiple of the group size
        return math.ceil(self.seq_len / self.world)

    @property
    def padded_seq(self) -> int:
        return self.local_seq * self.world

    @property
    def local_heads(self) -> int:
        assert self.num_heads % self.world == 0, "num_heads must be divisible by the sequence-parallel size"
        return self.num_heads // self.world

    @property
    def token_range(self) -> tuple[int, int]:
        return self.rank * self.local_seq, min((self.rank + 1) * self.local_seq, self.seq_len)

    # ---- first all-to-all: send buffer [dest][token][proj][local head][d] ----
    @property
    def send_row_stride(self) -> int:
        return self.n_proj * self.local_heads * self.head_dim

    @property
    def send_dest_stride(self) -> int:
        return self.local_seq * self.send_row_stride

    def qkv_col_offsets(self) -> torch.Tensor:
        """int64 [n_proj * H]: element offset (inside a send-buffer row group) of output column block j =
        proj * H + head of the fused QKV(+gate) GEMM."""
        Hl, d = self.local_heads, self.head_dim
        off = []
        for proj in range(self.n_proj):
            for h in range(self.num_heads):
                off.append((h // Hl) * self.send_dest_stride + proj * Hl * d + (h % Hl) * d)
        return torch.tensor(off, dtype=torch.int64)

    def push_col_offsets(self, peer_base: list, ref_base: int) -> torch.Tensor:
        """int64 [H]: for the push exchange (no send buffer): element offset, relative to `ref_base`, of head h of
        projection 0 in the receive buffer [padded_seq, n_proj, local_heads, d] of the rank that owns the head, at the
        first of MY token rows. peer_base / ref_base are byte addresses; rows advance by send_row_stride."""
        Hl, d = self.local_heads, self.head_dim
        first_row = self.rank * self.local_seq * self.send_row_stride
        off = []
        for h in range(self.num_heads):
            delta = peer_base[h // Hl] - ref_base
            assert delta % 16 == 0
            off.append(delta // 2 + first_row + (h % Hl) * d)
        return torch.tensor(off, dtype=torch.int64)

    def head_col_offsets(self) -> torch.Tensor:
        """int64 [H]: offsets of the heads of ONE projection (relative to that projection's base inside the send
        buffer) -- what the in-place RMSNorm/RoPE pass over q (and over k) needs."""
        Hl, d = self.local_heads, self.head_dim
        return torch.tensor([(h // Hl) * self.send_dest_stride + (h % Hl) * d for h in range(self.num_heads)],
                            dtype=torch.int64)


def pack_reference(x: torch.Tensor, plan: SPPlan) -> torch.Tensor:
    """Torch restatement of what fvb_linear_bf16_sp's column-block offsets do: x [local_seq, n_proj, H, d] ->
    send buffer [world, local_seq, n_proj, local_heads, d]. Only used by tests."""
    S, n, H, d = x.shape
    return x.view(S, n, plan.world, plan.local_heads, d).permute(2, 0, 1, 3, 4).contiguous()


def all_to_all_tokens_to_heads(send: torch.Tensor, group=None) -> torch.Tensor:
    """send [world, local_seq, ...] -> recv [world * local_seq, ...] (source-rank-major == global token order).
    sequence_model_parallel_all_to_all_4D(scatter heads, gather tokens), communication_op.py:28-32."""
    if send.shape[0] == 1:
        return send.view(send.shape[1], *send.shape[2:])
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv.view(send.shape[0], -1), send.view(send.shape[0], -1), group=group)
    return recv.view(send.shape[0] * send.shape[1], *send.shape[2:])


def all_to_all_heads_to_tokens(o: torch.Tensor, world: int, group=None) -> torch.Tensor:
    """o [world * local_seq, local_heads, d] (all tokens, my heads) -> recv [world(src), local_seq, local_heads, d]
    (my tokens, heads of every source rank; head index = src * local_heads + h)."""
    if world == 1:
        return o.view(1, *o.shape)
    send = o.view(world, -1)
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)
    return recv.view(world, o.shape[0] // world, *o.shape[1:])


# ----------------------------------------------------------------------------------------------------------------
# process-group plumbing
# ----------------------------------------------------------------------------------------------------------------
def init_from_env(backend: str | None = None):
    """Reads RANK / LOCAL_RANK / WORLD_SIZE / MASTER_* (torchrun). Returns (rank, world, device)."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if torch.cuda.is_available():
        torch.cuda.set_device(local)
        device = torch.device("cuda", local)
        backend = backend or "nccl"
    else:
        device = torch.device("cpu")
        backend = backend or "gloo"
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group(backend=backend, rank=rank, world_size=world,
                                device_id=device if backend == "nccl" else None)
    return rank, world, device


# ----------------------------------------------------------------------------------------------------------------
# sequence-parallel block / model forward (CUDA)
# ----------------------------------------------------------------------------------------------------------------
def out_proj_sp(back: torch.Tensor, blk, x: torch.Tensor, mod) -> torch.Tensor:
    """Self-attention out-projection + gated residual (epilogue and output dtype per the wan_dit.Modulation `mod`) of my
    S_loc tokens: the return buffer back [P(src), S_loc, Hl, d] is read in place as an A operand K-segmented by source rank."""
    from . import ops
    S_loc, D = x.shape
    seg = back.shape[2] * back.shape[3]
    y = torch.empty((S_loc, D), dtype=torch.bfloat16 if mod.bf16 else torch.float32, device=x.device)
    ops.linear_sp(back, S_loc, D, seg, blk.w_o, blk.b_o, y, D, mod.attn_epilogue, x_seg_len=seg, x_seg_stride=S_loc * seg,
                  resid=x, gate=mod.gate_msa, gate_rows=mod.rows)
    return y


class SPWanDiT:
    """WanDiT sharded over `world` ranks. Every rank holds all weights (replicated, as in the reference)."""

    def __init__(self, model, rank: int, world: int, group=None, comm: str | None = None):
        if model.cfg.fp8_linears:
            from ._lib import FvbError
            raise FvbError("sequence parallelism runs bf16 linears only: build the model with fp8_linears=False")
        if model.cfg.attention_8bit:
            from ._lib import FvbError
            raise FvbError("sequence parallelism runs bf16 attention only: build the model with attention_8bit=False")
        self.m = model
        self.rank, self.world, self.group = rank, world, group
        self._plans: dict = {}
        # "nccl": two all_to_all_single per layer on buffers the kernels fill / read in place.
        # "push": no all-to-all at all -- the RMSNorm/RoPE pass writes every head straight into the receive buffer of the
        #         rank that owns it (peer memory over NVLink, torch symmetric memory for the mapping and the barrier), and
        #         the attention output rows are copied to their token owners the same way.
        self.comm = comm or os.environ.get("FVB_SP_COMM", "push")
        self._push: dict = {}
        self._push_decision: bool | None = None  # set by the first forward, identically on every rank

    def _push_ok(self, plan: SPPlan, device) -> bool:
        """Decides ONCE, collectively, whether the symmetric-memory exchange is used: every rank attempts the set-up, the
        success flags are MIN-reduced over the group, and either all ranks push or all fall back to the NCCL all-to-all
        (a rank-local decision would leave some ranks in a symmetric-memory barrier and the others in all_to_all_single).
        Only the failures that mean "no peer mapping on this system" are absorbed; anything else is a bug and propagates."""
        if self._push_decision is not None:
            return self._push_decision
        ok, err = 1, None
        try:
            self._push_state(plan, device)
        except (ImportError, AttributeError, NotImplementedError, RuntimeError, torch.cuda.OutOfMemoryError) as e:
            ok, err = 0, e
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        self._push_decision = bool(flag.item())
        if not self._push_decision:
            self.comm = "nccl"
            self._push.clear()
            if self.rank == 0:
                import sys
                why = f"{type(err).__name__}: {err}" if err is not None else "another rank could not set it up"
                print(f"[fastvideo_b200] symmetric-memory exchange unavailable ({why}); every rank uses the NCCL all-to-all",
                      file=sys.stderr)
        return self._push_decision

    def _push_state(self, plan: SPPlan, device):
        """Symmetric receive buffers + offset table for one sequence length (allocated once; every rank must call this in
        the same order)."""
        key = plan.seq_len
        if key not in self._push:
            import torch.distributed._symmetric_memory as symm
            grp = self.group or dist.group.WORLD
            Hl, d = plan.local_heads, plan.head_dim
            recv = symm.empty((plan.padded_seq, plan.n_proj, Hl, d), dtype=torch.bfloat16, device=device)
            back = symm.empty((plan.world, plan.local_seq, Hl, d), dtype=torch.bfloat16, device=device)
            h_recv, h_back = symm.rendezvous(recv, grp), symm.rendezvous(back, grp)
            off = plan.push_col_offsets([int(p) for p in h_recv.buffer_ptrs], recv.data_ptr())
            # v (and gate) heads are written by the GEMM epilogue itself: column block j = (proj - 2) * H + head
            vg_off = torch.cat([off + p * Hl * d for p in range(2, plan.n_proj)]).to(device)
            off = off.to(device)
            peers_back = [h_back.get_buffer(r, (plan.world, plan.local_seq, Hl, d), torch.bfloat16) for r in range(plan.world)]
            # return path: my heads of rank r's tokens go to slot [me] of rank r's back buffer. The producing kernel
            # (VSA combine, or a row scatter after dense attention) stores there directly: table of the P destinations.
            seg = torch.tensor([peers_back[r][self.rank].data_ptr() for r in range(plan.world)], dtype=torch.int64, device=device)
            back.zero_()  # rows past seq_len in the last rank's slots are never written: they must read as zeros
            torch.cuda.synchronize(device)
            h_back.barrier(channel=1)
            self._push[key] = dict(recv=recv, back=back, h_recv=h_recv, h_back=h_back, off=off, vg_off=vg_off,
                                   peers_back=peers_back, seg=seg)
        return self._push[key]

    def plan(self, seq_len: int) -> SPPlan:
        cfg = self.m.cfg
        key = seq_len
        if key not in self._plans:
            p = SPPlan(self.world, self.rank, seq_len, cfg.num_attention_heads, cfg.head_dim, 4 if cfg.vsa else 3)
            dev = self.m.w_patch.device
            self._plans[key] = (p, p.qkv_col_offsets().to(dev), p.head_col_offsets().to(dev))
        return self._plans[key]

    def block_forward(self, x, blk, ctx, temb6, lay, plan_t, rope_row_local):
        from . import ops, vsa
        from .wan_dit import Modulation, block_tail, refuse_grad
        refuse_grad("SPWanDiT", blk, x, ctx, temb6)
        plan, qkv_off, head_off = plan_t
        cfg = self.m.cfg
        D, d, Hl, P = cfg.hidden_size, cfg.head_dim, plan.local_heads, self.world
        S_loc, S, S_pad, n_proj = plan.local_seq, plan.seq_len, plan.padded_seq, plan.n_proj
        mod = Modulation.fp32(blk, temb6)
        n1 = mod.norm1(x, cfg.eps)
        if self.comm == "push" and P > 1 and self._push_ok(plan, x.device):
            back = self._attention_push(n1, blk, lay, plan, rope_row_local)
        else:
            send = torch.empty((P, S_loc, n_proj, Hl, d), dtype=torch.bfloat16, device=x.device)
            ops.linear_sp(n1, S_loc, D, n1.stride(0), blk.w_qkv, blk.b_qkv, send, plan.send_row_stride, out_col_offsets=qkv_off)
            flat = send.view(-1)
            qb = flat.as_strided((S_loc, 1), (plan.send_row_stride, 1))
            kb = flat[Hl * d:].as_strided((S_loc, 1), (plan.send_row_stride, 1))
            ops.rmsnorm_rope_(qb, blk.norm_q, kb, blk.norm_k, lay.cos, lay.sin, rope_row_local, head_dim=d, eps=cfg.eps,
                              col_offsets=head_off, shape=(S_loc, D))
            recv = all_to_all_tokens_to_heads(send, self.group)  # [S_pad, n_proj, Hl, d]
            q = recv[:S, 0].unsqueeze(0)
            k = recv[:S, 1].unsqueeze(0)
            v = recv[:S, 2].unsqueeze(0)
            o = torch.zeros((1, S_pad, Hl, d), dtype=torch.bfloat16, device=x.device) if S_pad != S else \
                torch.empty((1, S_pad, Hl, d), dtype=torch.bfloat16, device=x.device)
            if cfg.vsa:
                vsa.video_sparse_attn_bshd(q, k, v, lay.vbs, lay.topk, gate=recv[:S, 3].unsqueeze(0), block_off=lay.block_off,
                                           row_block=lay.row_block, out=o[:, :S])
            else:
                ops.attention(q, k, v, softmax_scale=d ** -0.5, out=o[:, :S])
            back = all_to_all_heads_to_tokens(o[0], P, self.group)  # [P(src), S_loc, Hl, d]
        return block_tail(out_proj_sp(back, blk, x, mod), blk, ctx, mod, cfg)

    def _attention_push(self, n1, blk, lay, plan, rope_row_local):
        """Self-attention with the exchange done by peer-memory stores. Returns the return buffer [P, S_loc, Hl, d]."""
        from . import ops, vsa
        cfg = self.m.cfg
        D, d, Hl, P = cfg.hidden_size, cfg.head_dim, plan.local_heads, self.world
        S_loc, S, S_pad = plan.local_seq, plan.seq_len, plan.padded_seq
        st = self._push_state(plan, n1.device)
        recv, rs = st["recv"], plan.send_row_stride
        # v (and the VSA gate) need no normalisation: their GEMM's epilogue stores every head directly into the receive
        # buffer of the rank that owns it (column-block offsets reaching into peer memory), so that half of the exchange
        # rides on the GEMM tile by tile. q and k go to a local buffer first (RMSNorm is over the full row).
        ops.linear_sp(n1, S_loc, D, n1.stride(0), blk.w_qkv[2 * D:], blk.b_qkv[2 * D:], recv, rs, out_col_offsets=st["vg_off"])
        qk = ops.linear_any(n1, blk.w_qkv[:2 * D], blk.b_qkv[:2 * D])  # local [S_loc, 2D]
        base = recv.data_ptr()
        # q, k: RMSNorm + RoPE, every head written to its owner's receive buffer (projection p sits p*Hl*d further)
        ops.rmsnorm_rope_scatter(qk[:, :D], blk.norm_q, qk[:, D:], blk.norm_k, base, base + Hl * d * 2, rs, st["off"],
                                 lay.cos, lay.sin, rope_row_local, head_dim=d, eps=cfg.eps)
        st["h_recv"].barrier(channel=0)  # every rank's heads have landed here
        q, k, v = recv[:S, 0].unsqueeze(0), recv[:S, 1].unsqueeze(0), recv[:S, 2].unsqueeze(0)
        if cfg.vsa:
            # out = out_c * gate + out_s is written by the combine kernel straight into the token owners' buffers
            vsa.video_sparse_attn_bshd(q, k, v, lay.vbs, lay.topk, gate=recv[:S, 3].unsqueeze(0), block_off=lay.block_off,
                                       row_block=lay.row_block, out_segments=(st["seg"], S_loc, (0, Hl * d, d)))
        else:
            o = torch.empty((1, S, Hl, d), dtype=torch.bfloat16, device=n1.device)
            ops.attention(q, k, v, softmax_scale=d ** -0.5, out=o)
            ops.scatter_rows_to_segments(o[0].view(S, Hl * d), st["seg"], S_loc)
        st["h_back"].barrier(channel=1)
        return st["back"]

    @torch.no_grad()
    def forward(self, latents, text, timestep, vsa_sparsity=None):
        from . import ops
        m, cfg = self.m, self.m.cfg
        assert latents.shape[0] == 1, "sequence-parallel path runs one sample per forward"
        pt, ph, pw = cfg.patch_size
        seq_shape = (latents.shape[2] // pt, latents.shape[3] // ph, latents.shape[4] // pw)
        lay = m.layout(seq_shape, latents.device, vsa_sparsity if cfg.vsa else None)
        S = seq_shape[0] * seq_shape[1] * seq_shape[2]
        plan_t = self.plan(S)
        plan = plan_t[0]
        temb, tproj, ctx = m.condition(timestep, text)
        # patchify only this rank's tokens (sequence_model_parallel_shard, wanvideo.py:693)
        patches = m.patches(latents.to(torch.bfloat16))[0]
        lo, hi = plan.token_range
        order = lay.perm[lo:hi] if lay.perm is not None else torch.arange(lo, hi, device=latents.device)
        xl = torch.zeros((plan.local_seq, patches.shape[1]), dtype=torch.bfloat16, device=latents.device)
        xl[:hi - lo] = patches[order]
        x = ops.linear(xl, m.w_patch, m.b_patch)
        if hi - lo < plan.local_seq:
            x[hi - lo:] = 0  # the reference pads the embedded hidden states with zeros (communication_op.py:77-89)
        rope_row = torch.zeros(plan.local_seq, dtype=torch.int32, device=latents.device)
        rope_row[:hi - lo] = order.to(torch.int32)
        for blk in m.blocks:
            x = self.block_forward(x, blk, ctx[0], tproj[0:1], lay, plan_t, rope_row)
        y_loc = m.head(x, temb, lay, 0)  # [local_seq, C*pt*ph*pw]
        if self.world > 1:
            y = torch.empty((self.world, *y_loc.shape), dtype=y_loc.dtype, device=y_loc.device)
            dist.all_gather_into_tensor(y.view(-1), y_loc.contiguous().view(-1), group=self.group)
            y = y.view(-1, y_loc.shape[1])[:S]
        else:
            y = y_loc[:S]
        return m.unpatchify(y.unsqueeze(0), lay)

"""Data-parallel gradient exchange: rays shard across GPUs (one process per GPU), every rank holds a full
replica, and the parameter gradients are averaged once per step -- what the reference gets from Lightning DDP
(launch.py:98; SURVEY.md 8e).  NCCL over NVLink 5 / NVSwitch via torch.distributed; no data-path collective
other than this one exists on the path."""
import torch
import torch.distributed as dist


class GradSync:
    """comm_dtype=None: all-reduce the fp32 gradients as they are (what the reference's DDP does).
    comm_dtype=torch.bfloat16: large gradients (the hash table) travel as bf16 -- half the bytes on the wire, 8-bit mantissa;
    an opt-in wire-compression hook, not the default."""

    def __init__(self, params, world_size=None, group=None, comm_dtype=None, compress_min_numel=1 << 20):
        self.params = list(params)
        self.group = group
        self.world = world_size if world_size is not None else (dist.get_world_size(group) if dist.is_initialized() else 1)
        self.comm_dtype = comm_dtype
        self.compress_min_numel = compress_min_numel

    def all_reduce_mean(self):
        """in-place mean of every .grad over the ranks (largest tensor first so NCCL starts on the 50 MB
        hash-table gradient immediately)."""
        if self.world <= 1:
            return
        grads = [p.grad for p in self.params if p.grad is not None]
        grads.sort(key=lambda g: -g.numel())
        inv = 1.0 / self.world
        works, packed = [], []
        for g in grads:
            if self.comm_dtype is not None and g.numel() >= self.compress_min_numel:
                buf = g.to(self.comm_dtype)
                packed.append((g, buf))
                works.append(dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
            else:
                works.append(dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        for w in works:
            w.wait()
        for g, buf in packed:
            g.copy_(buf)
        for g in grads:
            g.mul_(inv)


def level_group_ranges(level_groups, level_offsets, table_first_float, n_total):
    """Pure host logic of P2PGradSync.bind_pipelined: the exchange range (begin, count) in floats of every level group.

    level_groups   ((l0, l1), ...) partitioning [0, L) from the top down, e.g. ((12, 16), (8, 12), (0, 8))
    level_offsets  entry offset of every level inside the table (L + 1 values, 2 floats per entry)
    table_first_float  index of the table's first float inside the exchange buffer (the table is the LAST parameter in it)
    n_total        length of the (padded) exchange buffer
    Group i covers the floats of its levels; the first group additionally runs to the end of the buffer (padding), the last one starts at 0
    (everything in front of the table: the other parameters and the density network's weights).  The ranges tile [0, n_total)."""
    groups = [tuple(g) for g in level_groups]
    L = len(level_offsets) - 1
    ok = groups and groups[0][1] == L and groups[-1][0] == 0 and all(groups[i][0] == groups[i + 1][1] for i in range(len(groups) - 1)) \
        and all(a < b for a, b in groups)
    if not ok or len(groups) > 4:
        raise ValueError(f'level_groups must partition [0, {L}) from the top down in at most 4 groups, e.g. ((12, 16), (8, 12), (0, 8))')
    off = lambda l: table_first_float + 2 * int(level_offsets[l])
    out = []
    for i, (l0, l1) in enumerate(groups):
        begin = 0 if i == len(groups) - 1 else off(l0)
        end = n_total if i == 0 else off(l1)
        if begin % 4 or end % 4 or end <= begin:
            raise ValueError('level group boundaries must be 16-byte aligned and non-empty')
        out.append((begin, end - begin))
    return out


class P2PGradSync:
    """The same mean, as OUR kernels over NVLink peer memory instead of NCCL (csrc/p2p.cu): the flat gradient vector of every rank
    lives in a symmetric (peer-mapped) buffer; ``all_reduce_mean`` = ONE kernel: entry barrier, in-place reduce-scatter + all-gather
    (rank r sums chunk r over the peers -- in the NVSwitch when the buffer has a multicast mapping -- and writes it into every replica),
    exit barrier.  ``bind_direct`` makes the fused backward accumulate straight into the buffer (no copy-in); afterwards ``p.grad`` IS the view of the symmetric buffer that holds the mean (no copy-out).
    Capturable into the step's CUDA graph (no NCCL call inside).  Needs torch.distributed._symmetric_memory (CUDA backend) and P2P
    access between the ranks' GPUs; ``make_grad_sync`` falls back to NCCL when that is not available."""

    def __init__(self, params, group=None):
        import ctypes
        import torch.distributed._symmetric_memory as symm
        self.params = [p for p in params if p.requires_grad and p.numel() > 0]
        self.params.sort(key=lambda p: p.numel())   # the hash table (largest) LAST: its level groups are then contiguous tails of the buffer
        if not self.params or not self.params[0].is_cuda:
            raise RuntimeError('P2PGradSync needs CUDA parameters')
        group = group if group is not None else dist.group.WORLD
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        dev = self.params[0].device
        if hasattr(symm, 'enable_symm_mem_for_group') and not symm.is_symm_mem_enabled_for_group(group.group_name):
            symm.enable_symm_mem_for_group(group.group_name)
        sizes = [(p.numel() + 3) // 4 * 4 for p in self.params]       # every slice 16-byte aligned
        self.n = (sum(sizes) + 4 * self.world - 1) // (4 * self.world) * (4 * self.world)   # equal float4 chunks per rank
        self.buf = symm.empty(self.n, dtype=torch.float32, device=dev)
        self.hdl = symm.rendezvous(self.buf, group)
        self.flags = symm.empty(256, dtype=torch.int32, device=dev)   # [0,16) nsr_p2p_barrier, channel c of nsr_p2p_exchange_mean_range [32 + 32 c, 64 + 32 c)
        self.fhdl = symm.rendezvous(self.flags, group)
        self.buf.zero_()
        self.flags.zero_()
        self.epoch = torch.zeros(1, dtype=torch.int32, device=dev)
        self.epoch2 = torch.zeros(4, 2, dtype=torch.int32, device=dev)   # one-launch exchange, per channel: {last completed epoch, CTA counter}
        self.ranges, self.side, self._pending = None, [], []
        self.direct = set()
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self.views, off = [], 0
        for p, sz in zip(self.params, sizes):
            self.views.append(self.buf[off:off + p.numel()].view_as(p))
            off += sz
        A = ctypes.c_uint64 * self.world
        self._peer = A(*[int(x) for x in self.hdl.buffer_ptrs])
        self._fpeer = A(*[int(x) for x in self.fhdl.buffer_ptrs])
        mc = int(getattr(self.hdl, 'multicast_ptr', 0) or 0)
        # NVSwitch multicast reduce (multimem.ld_reduce / multimem.st): NSR_P2P_MULTIMEM = 1 | 0 | auto.  At 2 ranks plain P2P
        # loads/stores beat the multicast mapping for the 50 MB exchange, so auto uses it only from 4 ranks up
        # (in-switch reduction moves 1/world of the bytes per GPU).
        import os
        # NSR_P2P_EXCHANGE = fused (default: barriers inside the one reduce kernel, nsr_p2p_exchange_mean) | legacy (barrier, reduce, barrier)
        self.one_launch = os.environ.get('NSR_P2P_EXCHANGE', 'fused') != 'legacy'
        want = os.environ.get('NSR_P2P_MULTIMEM', 'auto')
        use_mc = mc != 0 and (want == '1' or (want == 'auto' and self.world >= 4))
        self.multicast_available = mc != 0
        self.multicast = mc if use_mc else 0
        torch.cuda.synchronize()
        dist.barrier(group)   # every rank has zeroed its flags before anyone signals

    def view_of(self, param):
        """the slice of the symmetric buffer that holds (and after the exchange IS) this parameter's gradient"""
        for p, v in zip(self.params, self.views):
            if p is param:
                return v
        raise KeyError('parameter is not part of this exchange')

    def bind_direct(self, fused):
        """let the fused NeRF backward accumulate straight into the symmetric buffer (NerfFused.direct_grads): no 50 MB copy-in per step.
        The backward then zeroes + fills the views itself and autograd is bypassed for these two parameters."""
        if getattr(fused, 'contracted', False):
            raise ValueError('P2PGradSync.bind_direct / bind_pipelined serve the per-ray fused NeRF backward only; the unbounded (contracted, '
                             'two-pass) executor hands its gradients to autograd: exchange them with the NCCL GradSync instead')
        net, cnet = fused.net.params, fused.cnet.params
        fused.direct_grads = (self.view_of(net), self.view_of(cnet))
        self.direct = {id(net), id(cnet)}

    def bind_pipelined(self, fused, level_groups=((12, 16), (8, 12), (0, 8))):
        """bind_direct + overlap: the fused backward scatters the table gradient level group by level group (highest levels first) and calls
        ``exchange_group(i)`` behind each launch; the exchange of a finished group runs on a side stream beside the next group's scatter
        (the scatter launches leave one CTA slot per SM free for it), the last range -- everything below the first groups: the other
        parameters, the network weights, the coarse levels -- runs on the main stream, which then joins the side streams.
        What DDP does with gradient buckets (launch.py:98), for the one big tensor of this model."""
        self.bind_direct(fused)
        net = fused.net
        if self.params[-1] is not net.params:
            raise RuntimeError('bind_pipelined: the hash-grid parameter must be the largest parameter of the exchange')
        groups = [tuple(g) for g in level_groups]
        base = self.view_of(net.params).data_ptr() - self.buf.data_ptr()
        assert base % 16 == 0
        self.ranges = level_group_ranges(groups, fused.grid.offset, base // 4 + net.mlp.n_params, self.n)
        self.side = [torch.cuda.Stream(device=self.buf.device) for _ in groups[:-1]]
        fused.level_groups = groups
        fused.exchange_hook = self.exchange_group

    def exchange_group(self, i):
        """exchange of range i (called by the backward right behind the scatter launch of level group i)"""
        import ctypes
        from .lib import lib, ptr
        mc = ctypes.c_void_p(self.multicast) if self.multicast else None
        begin, count = self.ranges[i]
        cur = torch.cuda.current_stream()
        last = i == len(self.ranges) - 1
        st = cur if last else self.side[i]
        if not last:
            st.wait_stream(cur)
        lib.call('nsr_p2p_exchange_mean_range', self._peer, self._fpeer, mc, ptr(self.epoch2[i]), ptr(self.err), self.rank, self.world, begin, count,
                 i, 1 if not last else 0, ctypes.c_void_p(st.cuda_stream))
        if last:
            for sd in self.side:
                cur.wait_stream(sd)
            for p, v in zip(self.params, self.views):
                p.grad = v

    def finish(self):
        """post-backward hook of the pipelined mode: the exchanges were launched from inside the backward; gradients are the views"""
        for p, v in zip(self.params, self.views):
            p.grad = v

    def all_reduce_mean(self):
        import ctypes
        from .lib import lib, ptr, stream
        for p, v in zip(self.params, self.views):
            if id(p) in self.direct:
                continue   # the backward kernels accumulated into the view already
            if p.grad is None:
                v.zero_()
            elif p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
        mc = ctypes.c_void_p(self.multicast) if self.multicast else None
        if self.one_launch:
            lib.call('nsr_p2p_exchange_mean', self._peer, self._fpeer, mc, ptr(self.epoch2[0]), ptr(self.err), self.rank, self.world, self.n, stream())
        else:
            bar = lambda: lib.call('nsr_p2p_barrier', self._fpeer, ptr(self.epoch), ptr(self.err), self.rank, self.world, stream())
            bar()
            lib.call('nsr_p2p_allreduce_mean', self._peer, mc, self.rank, self.world, self.n, stream())
            bar()
        for p, v in zip(self.params, self.views):
            p.grad = v

    def self_test(self, group=None):
        """one exchange of a rank-dependent pattern, compared with torch.distributed's all-reduce; False => do not use this path."""
        saved = [p.grad for p in self.params]
        try:
            gen = torch.Generator(device=self.buf.device).manual_seed(1234 + self.rank)
            pat = [torch.randn(p.shape, device=p.device, generator=gen) for p in self.params]
            ref = [x.clone() for x in pat]
            for r in ref:
                dist.all_reduce(r, group=group)
                r.div_(self.world)
            for p, x in zip(self.params, pat):
                p.grad = x
            self.all_reduce_mean()
            torch.cuda.synchronize()
            ok = int(self.err.item()) == 0 and all(bool(torch.allclose(p.grad, r, rtol=1e-5, atol=1e-6)) for p, r in zip(self.params, ref))
        except Exception:
            ok = False
        flag = torch.tensor([1 if ok else 0], device=self.buf.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)   # every rank takes the same decision
        for p, g in zip(self.params, saved):
            p.grad = g
        return bool(flag.item())

    def check(self):
        """host-side check of the device error flag (a peer that never reached a barrier); one sync."""
        if int(self.err.item()) != 0:
            raise RuntimeError('P2PGradSync: a peer did not reach the barrier within the spin bound')


def make_grad_sync(params, world, group=None, comm_dtype=None, prefer_p2p=True):
    """-> (sync object with .all_reduce_mean(), description).  P2P kernels over NVLink when available, NCCL otherwise."""
    params = list(params)
    if world > 1 and prefer_p2p and comm_dtype is None and params and params[0].is_cuda:
        try:
            s = P2PGradSync(params, group)
            if not s.self_test(group):
                return GradSync(params, world, group, comm_dtype), 'NCCL all-reduce (p2p self-test failed)'
            return s, 'nsr p2p kernels over NVLink peer memory' + (' (NVSwitch multicast reduce)' if s.multicast else ' (P2P loads/stores)')
        except Exception as e:  # symmetric memory / P2P mapping unavailable: NCCL does the same exchange
            why = f'{type(e).__name__}: {e}'.splitlines()[0][:160]
            return GradSync(params, world, group, comm_dtype), f'NCCL all-reduce (p2p unavailable: {why})'
    return GradSync(params, world, group, comm_dtype), 'NCCL all-reduce' + (f' ({comm_dtype})' if comm_dtype is not None else '')


def shard_rays(rays, rank, world):
    """contiguous shard of a [N, 6] ray batch for this rank (N divisible by world, SURVEY 8e: 65,536 / 8)."""
    n = rays.shape[0] // world
    return rays[rank * n:(rank + 1) * n]

"""Frame sharding of one clip over the GPUs of a box (SURVEY.md 8e).

Where the path shards: with `reset_branch = R` the forward recurrence restarts every R calls
(RefVSR.py:168-170), and a restarted call depends on nothing but its own window; the backward branch is
window-local (RefVSR.py:211-214).  Hence output frames [sR, (s+1)R) form independent *segments*
(verified bit-exact against the reference: SURVEY appendix B) and a clip splits over ranks at segment
boundaries with NO collective on the data path.  The only exchange is an *input halo*: a rank that owns
(decoded / received) frames [f0, f1) needs T//2 neighbour frames on each side to build its first and last
windows.  `exchange_halo` moves exactly those frames with point-to-point send/recv (NCCL over NVLink on the
GPU box, gloo in the CPU tests).  Results can be gathered to rank 0 with `gather_frames`.

`reset_branch = None` (the 8K configs) has no segment boundaries: the forward chain is serial, and the
honest multi-GPU mode is independent replicas over different clips.
"""
import torch
import torch.distributed as dist


def plan_segments(num_frames, reset_branch, world_size):
    """-> list over ranks of (f0, f1): contiguous, reset-aligned ownership ranges covering [0, num_frames)."""
    if reset_branch is None:
        raise ValueError('reset_branch=None: the forward recurrence never restarts, a clip cannot be frame-sharded '
                         '(run independent replicas over different clips instead)')
    nseg = (num_frames + reset_branch - 1) // reset_branch
    per, extra = divmod(nseg, world_size)
    out, s = [], 0
    for r in range(world_size):
        n = per + (1 if r < extra else 0)
        out.append((min(s * reset_branch, num_frames), min((s + n) * reset_branch, num_frames)))
        s += n
    return out


def exchange_halo(local, plan, rank, halo, group=None):
    """`local`: frames owned by this rank, shape (f1-f0, ...).  Returns (frames, first_index) where `frames`
    additionally holds up to `halo` frames from the neighbouring ranks on each side."""
    world = len(plan)
    f0, f1 = plan[rank]
    num_frames = plan[-1][1]
    if f1 <= f0:                      # a rank that owns nothing neither sends nor receives (its neighbours skip it, too)
        return local, f0
    lo, hi = max(f0 - halo, 0), min(f1 + halo, num_frames)
    parts = {}
    ops, keep = [], []
    for other in range(world):
        if other == rank:
            continue
        o0, o1 = plan[other]
        # frames I need from `other`
        a, b = max(lo, o0), min(hi, o1)
        if a < b and (a < f0 or b > f1) and o1 > o0:
            a2, b2 = (a, min(b, f0)) if a < f0 else (max(a, f1), b)
            buf = torch.empty((b2 - a2,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
            parts[a2] = buf
            ops.append(dist.P2POp(dist.irecv, buf, other, group))
        # frames `other` needs from me
        olo, ohi = max(o0 - halo, 0), min(o1 + halo, num_frames)
        a, b = max(olo, f0), min(ohi, f1)
        if a < b and (a < o0 or b > o1) and o1 > o0:
            a2, b2 = (a, min(b, o0)) if a < o0 else (max(a, o1), b)
            if a2 < b2:
                snd = local[a2 - f0:b2 - f0].contiguous()
                keep.append(snd)
                ops.append(dist.P2POp(dist.isend, snd, other, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    parts[f0] = local
    frames = torch.cat([parts[k] for k in sorted(parts)], 0) if len(parts) > 1 else local
    return frames, lo


def run_sharded(net, frames_lr, frames_ref, first_index, own, num_frames, T):
    """Process the owned output frames `own = (f0, f1)`.  `frames_*` hold clip frames
    [first_index, first_index + len) (own + halo).  Yields (k, result (3, scale*h, scale*w)).  The first owned frame
    starts a new stream (is_first_frame=True) - it sits on a reset boundary by construction."""
    f0, f1 = own
    for k in range(f0, f1):
        idx = [min(max(k - T // 2 + j, 0), num_frames - 1) - first_index for j in range(T)]   # datasets.py:233-234
        assert min(idx) >= 0 and max(idx) < frames_lr.shape[0], 'halo too small for the window'
        sel = torch.tensor(idx, device=frames_lr.device)
        out = net(frames_lr.index_select(0, sel).unsqueeze(0), frames_ref.index_select(0, sel).unsqueeze(0),
                  k == f0, False, False)['result']
        yield k, out[0]


def gather_frames(results, plan, rank, shape, device, dtype=torch.float32, group=None):
    """all ranks -> rank 0: list of num_frames tensors (rank 0) or None.  Uses all_gather on padded blocks
    (works with both NCCL and gloo)."""
    world = len(plan)
    mx = max(b - a for a, b in plan)
    mine = torch.zeros((mx,) + tuple(shape), dtype=dtype, device=device)
    for i, (k, r) in enumerate(sorted(results)):
        mine[i].copy_(r)
    bufs = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(bufs, mine, group=group)
    if rank != 0:
        return None
    out = []
    for r, (a, b) in enumerate(plan):
        out.extend(bufs[r][i] for i in range(b - a))
    return out


# ------------------------------------------------------------------------------------------------------------------
# BASELINE configs[3]: ONE clip sharded by FRAMES over the GPUs of a box, finer than the reset segments (SURVEY 8e)
# ------------------------------------------------------------------------------------------------------------------
def plan_frames(num_frames, world_size):
    """contiguous, balanced ownership ranges (no alignment to reset_branch): 32 frames / 8 ranks -> 4 frames each"""
    per, extra = divmod(num_frames, world_size)
    out, s = [], 0
    for r in range(world_size):
        n = per + (1 if r < extra else 0)
        out.append((s, s + n))
        s += n
    return out


def chain_pieces(own, reset_branch):
    """Split an ownership range at the chain heads (frames k with k % reset_branch == 0, where the forward recurrence
    restarts from zeros, RefVSR.py:168-170) -> [(k0, k1, is_head)].  Only the first piece can need an incoming state."""
    f0, f1 = own
    cuts = [f0] + [k for k in range(f0 + 1, f1) if k % reset_branch == 0] + [f1]
    return [(a, b, a % reset_branch == 0) for a, b in zip(cuts[:-1], cuts[1:]) if a < b]


def _pack_state(state, buf):
    o = 0
    for t in state:
        nb = t.numel() * t.element_size()
        buf[o:o + nb].copy_(t.reshape(-1).view(torch.uint8))
        o += nb


def _unpack_state(buf, state):
    o = 0
    for t in state:
        nb = t.numel() * t.element_size()
        t.reshape(-1).view(torch.uint8).copy_(buf[o:o + nb])
        o += nb


def run_clip_frame_sharded(net, frames_lr, frames_ref, g0, plan, rank, groups=None, pre_windows=None, timing=None):
    """Process this rank's frames of ONE clip; returns [(k, (3, scale*h, scale*w) tensor)] in frame order.

    `frames_*`: clip frames [g0, g0 + m) = own range + T//2 input halo on each side (exchange_halo), on the compute device.
    Work split (DESIGN.md section 6):
      * local, embarrassingly parallel: per-frame products (flows, matching, reference features / alignment), the
        window-local backward branch (4 of the 5 propagation steps of a frame at T = 7) and the upsampling tail;
      * serial across ranks: the forward-branch step of frame k needs the state after frame k-1.  The chain restarts at
        every multiple of reset_branch, so a 32-frame clip has 4 independent chains.  A rank first runs the pieces of its
        range that START a chain (no input needed) and sends the state on; then it fills the wait for its predecessor with
        local windows whose forward step is done (default: until the message has landed; `pre_windows`: a fixed count), receives {feat (h,w,C), featUP (2h,2w,C),
        conf (h,w)} = (5C + 1) * P elements (62 MB in bf16 at 270x480) with ONE point-to-point message, runs its steps,
        sends the state on, and finishes its remaining windows.  The flow that warps the received state is a pure function
        of two input frames the rank already holds (halo), so it is recomputed, not sent.
    `groups`: optional pair of process groups; the transfer r -> r+1 uses groups[r % 2] so that a rank's send and receive
    never queue behind each other on one communicator stream.  `timing`: dict that receives the host-side phase list."""
    net_ = net.Network if hasattr(net, 'Network') else net
    world = len(plan)
    own = plan[rank]
    num_frames = plan[-1][1]
    R = net_.max_frame_itr_num
    T = net_.config.frame_num
    if own[1] <= own[0]:
        return []
    pieces = chain_pieces(own, R)
    need_recv = not pieces[0][2]
    f1 = own[1]
    need_send = f1 < num_frames and f1 % R != 0
    net_.shard_begin(frames_lr, frames_ref, g0, own, num_frames)
    try:
        dev = frames_lr.device
        st_in = net_.shard_state_buffers('in')
        nbytes = sum(t.numel() * t.element_size() for t in st_in)
        msg_in = net_._buf('sh.msg_in', (nbytes,), torch.uint8)
        msg_out = net_._buf('sh.msg_out', (nbytes,), torch.uint8)
        grp = (lambda r: None) if groups is None else (lambda r: groups[r % 2])
        work_recv = work_send = None
        if need_recv:                                     # posted up front: the message lands whenever the predecessor is done
            work_recv = dist.irecv(msg_in, src=rank - 1, group=grp(rank - 1))
        results, done = {}, set()
        log = []

        def finish(k):
            results[k] = net_.shard_finish_window(k)
            done.add(k)
            log.append(('window', k))

        def forward(k0, k1, head):
            nonlocal work_send
            state = None
            if not head:
                work_recv.wait()                          # NCCL: the compute stream waits for the transfer; gloo: host blocks
                _unpack_state(msg_in, st_in)
                state = st_in
                log.append(('recv', rank - 1))
            out_state = net_.shard_forward_piece(k0, k1, state)
            log.append(('forward', k0, k1, head))
            if k1 == f1 and need_send:
                _pack_state(out_state, msg_out)
                work_send = dist.isend(msg_out, dst=rank + 1, group=grp(rank))
                log.append(('send', rank + 1))

        # 1. pieces that start a chain need no input: run them first so the successor can start early
        for k0, k1, head in pieces:
            if head:
                forward(k0, k1, True)
        if need_recv:
            k0, k1, _ = pieces[0]
            net_.shard_prefetch_forward(k0, k1, False)    # state-independent products of the dependent piece
            # 2. fill the wait for the predecessor with local windows whose forward step is already done
            ready = [k for k in range(own[0], own[1]) if k in net_._shard['fw_out']]
            if pre_windows is None:
                # dynamic: keep finishing local windows until the predecessor's message has landed (the completion poll is a
                # host-side event query; one host sync per window keeps the decision tied to real time)
                for k in ready:
                    if work_recv.is_completed():
                        break
                    finish(k)
                    if dev.type == 'cuda':
                        torch.cuda.current_stream(dev).synchronize()
            else:
                for k in ready[:pre_windows]:
                    finish(k)
            forward(k0, k1, False)
        # 3. everything else
        for k in range(own[0], own[1]):
            if k not in done:
                finish(k)
        if work_send is not None:
            work_send.wait()
        if timing is not None:
            timing['log'] = log
        return [(k, results[k]) for k in sorted(results)]
    finally:
        net_.shard_end()

"""Multi-GPU plumbing for the decode path (one process per GPU): frames shard f % world, the only exchange is the hand-over
of the decoded fountain chunk records to rank 0 -- the role of concurrent_fountain_decoder_sink in the reference
(src/lib/fountain/concurrent_fountain_decoder_sink.h:58-84).

The exchange itself lives behind the C ABI (include/cb200.h, csrc/gather.cu); torch.distributed is only the host channel
that carries the 64-byte IPC handle / the 128-byte NCCL id between the processes at start-up:

  RecordExchange(ctx, "window")  every rank's RS / chunk-mask kernels store straight into a window in rank 0's HBM over NVLink
                                 (CUDA IPC peer mapping); epochs are published / awaited with system-scope flags on the device
  RecordExchange(ctx, "nccl")    cb200_gather_chunks: ncclSend / ncclRecv on a side stream, overlapping the next decode
  gather_records(...)            plain torch.distributed.gather of host or device tensors (gloo in the CPU tests)
"""
import torch
import torch.distributed as dist


def shard_frames(n_frames, rank, world):
    """frame f belongs to rank f % world (SURVEY 8e): indices of this rank's frames"""
    return list(range(rank, n_frames, world))


def gather_records(chunks, mask, dst=0):
    """chunks: (n, chunks_per_frame*chunk_size) uint8, mask: (n,) int32 -- same n on every rank.
    Returns (list_of_chunks, list_of_masks) on dst, (None, None) elsewhere."""
    world = dist.get_world_size()
    rank = dist.get_rank()
    gc = [torch.empty_like(chunks) for _ in range(world)] if rank == dst else None
    gm = [torch.empty_like(mask) for _ in range(world)] if rank == dst else None
    dist.gather(chunks, gc, dst=dst)
    dist.gather(mask, gm, dst=dst)
    return gc, gm


class RecordExchange:
    """Double-buffered hand-over of `n` chunk records per rank and step to rank 0.

    step s (1, 2, 3, ...) uses buffer s & 1:
        d_chunks, d_mask = ex.begin(s)        # where this rank's decode of step s must write (device addresses)
        ctx.decode_chunks_dev(frames, n, d_chunks, d_mask, ...)
        ex.end(s)                             # publish / start the exchange of step s
        ... on rank 0, whenever the records of step s are needed (typically one step later, so that the exchange overlaps
        the next decode):  ex.collect(s) -> (d_all_chunks, d_all_masks) device addresses, rank-major, valid on the context's
        stream; ex.release(s) when rank 0 is done with them."""

    def __init__(self, ctx, kind, n, rank=None, world=None):
        import libcimbar_b200 as cb
        self.ctx, self.kind, self.n = ctx, kind, n
        self.rank = dist.get_rank() if rank is None else rank
        self.world = dist.get_world_size() if world is None else world
        info = ctx.info
        self.rec_bytes = info.data_bytes
        self.send = None
        if kind in ("window", "window-direct"):
            box = [ctx.gather_root_create(self.world) if self.rank == 0 else None]
            dist.broadcast_object_list(box, src=0)
            if self.rank != 0:
                ctx.gather_peer_open(self.world, self.rank, box[0])
                if kind == "window":       # push form: the decode writes locally, a copy engine moves the records to rank 0
                    dev = torch.device("cuda", torch.cuda.current_device())
                    self.send = [(torch.empty((n, self.rec_bytes), dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
                                 for _ in range(2)]
        elif kind == "nccl":
            box = [cb.comm_unique_id() if self.rank == 0 else None]
            dist.broadcast_object_list(box, src=0)
            ctx.comm_init(box[0], self.world, self.rank)
            dev = torch.device("cuda", torch.cuda.current_device())
            self.send = [(torch.empty((n, self.rec_bytes), dtype=torch.uint8, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
                         for _ in range(2)]
            self.recv = [(torch.empty((self.world, n, self.rec_bytes), dtype=torch.uint8, device=dev),
                          torch.empty((self.world, n), dtype=torch.int32, device=dev)) if self.rank == 0 else (None, None)
                         for _ in range(2)]
        else:
            raise ValueError("kind must be 'window', 'window-direct' or 'nccl'")

    def begin(self, step):
        b = step & 1
        if self.kind == "window" and self.rank != 0:
            if step > 2:
                self.ctx.gather_chunks_wait(b)                 # the transfer of step - 2 out of these local buffers is done
            c, m = self.send[b]
            return c.data_ptr(), m.data_ptr()
        if self.kind in ("window", "window-direct"):
            if step > 2:
                self.ctx.gather_acquire(b, step - 2)           # rank 0 has let go of the records of step - 2
            return self.ctx.gather_slot(b)
        if step > 2:
            self.ctx.gather_chunks_wait(b)                     # the send buffers of step - 2 are free again (side stream done)
        c, m = self.send[b]
        return c.data_ptr(), m.data_ptr()

    def end(self, step):
        b = step & 1
        if self.kind == "window" and self.rank != 0:
            c, m = self.send[b]
            self.ctx.gather_push(b, c.data_ptr(), m.data_ptr(), self.n, step, step - 2 if step > 2 else 0)
        elif self.kind in ("window", "window-direct"):
            self.ctx.gather_publish(b, step)
        else:
            c, m = self.send[b]
            ac, am = self.recv[b]
            self.ctx.gather_chunks(self.world, self.rank, b, c.data_ptr(), m.data_ptr(), self.n,
                                   ac.data_ptr() if ac is not None else None, am.data_ptr() if am is not None else None)

    def collect(self, step):
        """rank 0: make the context's stream wait for every rank's records of `step`; returns their device addresses"""
        b = step & 1
        if self.kind in ("window", "window-direct"):
            self.ctx.gather_wait(b, step)
            return self.ctx.gather_slot(b, 0)                  # rank r's records: + r * slot stride (ctx.gather_slot(b, r))
        self.ctx.gather_chunks_wait(b)
        ac, am = self.recv[b]
        return ac.data_ptr(), am.data_ptr()

    def release(self, step):
        if self.kind in ("window", "window-direct") and self.rank == 0:
            self.ctx.gather_release(step & 1, step)


def stripe(n_total, rank, n_per_rank):
    """rank's contiguous stripe [start, stop) of a batch of n_total pictures, n_per_rank per rank (rank-major = batch order): the
    last ranks of a short batch get a short or an empty stripe"""
    start = min(n_total, rank * n_per_rank)
    return start, min(n_total, start + n_per_rank)


class CameraExchange:
    """Camera batches across ranks: every step, rank r decodes the contiguous stripe of the batch that `stripe` gives it (at most
    n_per_rank pictures) into the record window of RecordExchange ("window": local buffers + copy-engine push, "window-direct": the
    decode stores into rank 0's window), and rank 0 collects the records, masks and extract statuses of all ranks in batch order.

    With CB200_FLAG_CC_FIT in `flags` the ranks' contexts are linked to a CCM chain (cb200_ccm_chain_*), so that the colour
    decisions, chunks and masks equal those of one context decoding the whole batch:

        ex = CameraExchange(ctx, "window", n_per_rank, flags=cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT)
        for s in 1, 2, ...:
            ex.decode(s, ("rgb", d_pictures, wh))     # or ("jpeg", files) / ("png", files): this rank's stripe (may be empty)
            out = ex.collect(s)                      # every rank calls it; rank 0: (chunks, masks, statuses) as numpy, else None

    decode() only enqueues work; collect() synchronises the context's stream."""

    def __init__(self, ctx, kind, n_per_rank, flags=0, rank=None, world=None):
        import libcimbar_b200 as cb
        import torch
        if kind not in ("window", "window-direct"):
            raise ValueError("kind must be 'window' or 'window-direct'")
        self.ctx, self.kind, self.n, self.flags = ctx, kind, n_per_rank, flags
        self.rank = dist.get_rank() if rank is None else rank
        self.world = dist.get_world_size() if world is None else world
        self.records = RecordExchange(ctx, kind, n_per_rank, self.rank, self.world)
        self.chained = bool(flags & cb.FLAG_CC_FIT)
        if self.chained:
            box = [ctx.ccm_chain_root_create(self.world) if self.rank == 0 else None]
            dist.broadcast_object_list(box, src=0)
            if self.rank != 0:
                ctx.ccm_chain_peer_open(self.world, self.rank, box[0])
            ctx.ccm_chain_attach(self.rank, self.world)
        dev = torch.device("cuda", torch.cuda.current_device())
        self.status = [torch.zeros(max(1, n_per_rank), dtype=torch.int32, device=dev) for _ in range(2)]
        self.counts = {}

    def decode(self, step, batch):
        """enqueue the decode of this rank's stripe for `step` (1, 2, ...): batch = ("rgb", d_pictures, wh) with wh an (n, 2) array
        of (width, height) of the pictures packed in device memory, or ("jpeg" | "png", list of files as bytes)"""
        kind = batch[0]
        n = len(batch[2]) if kind == "rgb" else len(batch[1])
        if n > self.n:
            raise ValueError(f"{n} pictures in a stripe of {self.n}")
        self.counts[step] = n
        d_chunks, d_mask = self.records.begin(step)
        d_status = self.status[step & 1].data_ptr()
        if self.chained:
            self.ctx.ccm_chain_step(step)
        if kind == "rgb":
            # (an empty stripe still makes the call -- its part of the CCM chain -- with a stand-in address that is never read)
            self.ctx.scan_extract_decode_chunks_dev(batch[1] if n else d_status, batch[2], d_chunks, d_mask, d_status, flags=self.flags)
        elif kind == "jpeg":
            self.ctx.jpeg_scan_extract_decode_chunks_dev(batch[1], d_chunks, d_mask, d_status, flags=self.flags)
        elif kind == "png":
            self.ctx.png_scan_extract_decode_chunks_dev(batch[1], d_chunks, d_mask, d_status, flags=self.flags)
        else:
            raise ValueError("batch kind must be 'rgb', 'jpeg' or 'png'")
        self.records.end(step)

    def collect(self, step):
        """collective: rank 0 returns (chunks (n, data_bytes) uint8, masks (n,) uint32, statuses (n,) int32) of the whole batch of
        `step` in batch order, the other ranks None.  Synchronises the context's stream; raises if a rank of the exchange or of the
        CCM chain did not arrive in time"""
        import ctypes as C
        import numpy as np
        n = self.counts.pop(step)
        b = step & 1
        if self.rank == 0:
            self.records.collect(step)
        self.ctx.sync()
        if self.chained:
            self.ctx.ccm_chain_status()
        mine = (n, self.status[b][:n].cpu().numpy())
        parts = [None] * self.world if self.rank == 0 else None
        dist.gather_object(mine, parts, dst=0)
        if self.rank != 0:
            return None
        self.ctx.gather_status()
        cudart = C.CDLL("libcudart.so.12")
        rec = self.ctx.info.data_bytes
        chunks, masks, statuses = [], [], []
        for r, (nr, st) in enumerate(parts):
            pc, pm = self.ctx.gather_slot(b, r)
            hc = np.zeros((nr, rec), np.uint8)
            hm = np.zeros(nr, np.uint32)
            if nr:
                assert cudart.cudaMemcpy(C.c_void_p(hc.ctypes.data), C.c_void_p(pc), C.c_size_t(nr * rec), 2) == 0
                assert cudart.cudaMemcpy(C.c_void_p(hm.ctypes.data), C.c_void_p(pm), C.c_size_t(4 * nr), 2) == 0
            chunks.append(hc); masks.append(hm); statuses.append(st)
        self.records.release(step)
        return np.concatenate(chunks), np.concatenate(masks), np.concatenate(statuses)

"""Batch-parallel multi-GPU inference: images shard across ranks (one process per
GPU, torch.distributed over NCCL/NVLink); weights are replicated (seeded init or
broadcast); the only data-path collective is ONE all-gather of the fixed-size
detection records per batch (SURVEY.md section 8e).  The reference itself is
single-device (SSD300.py:458-462)."""
import os

import numpy as np
import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Reads RANK / WORLD_SIZE / LOCAL_RANK / MASTER_* (torchrun)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if torch.cuda.is_available():
        torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        dist.init_process_group(backend or ("nccl" if torch.cuda.is_available() else "gloo"),
                                rank=rank, world_size=world)
    return rank, world, local


def shard_range(total, rank, world):
    """Contiguous shard: rank r takes images [r*B/G, (r+1)*B/G)."""
    assert total % world == 0, "global batch must divide evenly across ranks"
    per = total // world
    return rank * per, (rank + 1) * per


_CTX = {"ctx": None, "failed": False}


def cabi_ctx():
    """The C-ABI communicator (odt_ctx: one NCCL communicator per process, include/odt_b200.h) over the ranks of the
    default torch.distributed group, created on first use: rank 0's 128-byte id travels through torch.distributed.
    None when it cannot be used (CPU-only process, ODT_COLLECTIVES=torch, NCCL not loadable) -- the collectives
    then go through torch.distributed."""
    if _CTX["ctx"] is not None or _CTX["failed"]:
        return _CTX["ctx"]
    # ODT_COLLECTIVES=torch is the functional fallback for hosts where NCCL cannot be loaded through the C ABI
    if (os.environ.get("ODT_COLLECTIVES", "cabi") == "torch" or not torch.cuda.is_available()
            or not dist.is_initialized() or dist.get_world_size() == 1):
        _CTX["failed"] = True
        return None
    import ctypes as C
    from . import lib as L
    lib = L.load()
    rank, world = dist.get_rank(), dist.get_world_size()
    buf = C.create_string_buffer(128)
    rc = lib.odt_ctx_unique_id(buf) if rank == 0 else 0
    box = [bytes(buf.raw) if rc == 0 else None]
    dist.broadcast_object_list(box, src=0)     # every rank learns whether rank 0 has NCCL, and the id
    if box[0] is None:
        _CTX["failed"] = True
        return None
    ctx = C.c_void_p()
    rc = lib.odt_ctx_create(C.byref(ctx), rank, world, box[0])
    ok = torch.tensor([1 if rc == 0 else 0], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)   # all ranks take the same route
    if int(ok.item()) != 1:
        if rc == 0:
            lib.odt_ctx_destroy(ctx)
        _CTX["failed"] = True
        return None
    _CTX["ctx"] = ctx
    return ctx


def gather_records(rec, group=None, out=None):
    """ONE all-gather of the packed per-image records [B, D*6+2] (written by the NMS kernel itself, see
    engine.Tail) on the current stream; returns [world*B, D*6+2] on every rank (`out`: preallocated destination).
    CUDA tensors of the default group go through the C ABI (odt_allgather_dets), everything else -- gloo on CPU,
    sub-groups -- through torch.distributed."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return rec
    if out is None:
        out = torch.empty((world * rec.shape[0], rec.shape[1]), dtype=rec.dtype, device=rec.device)
    ctx = cabi_ctx() if (rec.is_cuda and group is None and rec.is_contiguous() and rec.dtype == torch.float32) else None
    if ctx is not None:
        from . import lib as L
        L.check(L.load().odt_allgather_dets(ctx, rec.data_ptr(), out.data_ptr(), rec.numel(),
                                            torch.cuda.current_stream().cuda_stream), "allgather_dets")
        return out
    dist.all_gather_into_tensor(out, rec, group=group)
    return out


def broadcast_weights(weights, src=0):
    """Replicate rank `src`'s variables (name -> ndarray) to every rank: one flat fp32 buffer, one broadcast
    (odt_bcast_weights through the C ABI on GPUs, torch.distributed otherwise)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return weights
    dev = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
    names = sorted(weights)
    arrs = [np.ascontiguousarray(weights[k], dtype=np.float32) for k in names]
    flat = torch.from_numpy(np.concatenate([a.reshape(-1) for a in arrs]) if arrs else np.zeros(0, np.float32)).to(dev)
    ctx = cabi_ctx() if dev.type == "cuda" else None
    if ctx is not None and flat.numel():
        from . import lib as L
        L.check(L.load().odt_bcast_weights(ctx, flat.data_ptr(), flat.numel() * 4, src,
                                           torch.cuda.current_stream().cuda_stream), "bcast_weights")
    else:
        dist.broadcast(flat, src)
    host = flat.cpu().numpy()
    out, off = {}, 0
    for k, a in zip(names, arrs):
        out[k] = host[off:off + a.size].reshape(a.shape).copy()
        off += a.size
    return out


def detect_sharded(model, images_local, consumer=None):
    """Run this rank's image shard and all-gather everybody's detection records.  consumer=None: every
    rank reads back and returns all ranks' detections; consumer=r: only rank r does (the others return
    their own shard's detections)."""
    from .api import _as_host_tensor
    from .engine import unpack_records
    images_local = _as_host_tensor(images_local)
    net = model.engine(images_local.shape[0])
    net.image_buf.copy_(images_local, non_blocking=True)
    net.run()
    rec = gather_records(net.tail.rec)
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world > 1 and consumer is not None and dist.get_rank() != consumer:
        rec = net.tail.rec
    return unpack_records(rec.cpu().numpy(), net.tail.p.cap)

"""Multi-GPU determinism on hardware (SURVEY §4 "same image regardless of rank count"; VERDICT r1 item 7): needs >= 2 GPUs,
skipped on a 1-GPU machine. World 2: one process per GPU, weights from rank 0 through the library's own NCCL
broadcast (sdb_broadcast_weights), images sharded i mod world. Image i must be BIT-identical to what a 1-rank run produces."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_IMAGES, STEPS, HL = 4, 3, 32


def _sample(ctx, i):
    from stable_diffusion_burn_b200 import parallel, synth
    c = synth.make_context(1, 9, seed=500 + i)
    unc = synth.make_context(1, 2, seed=99)[0]
    lat = synth.make_latent(1, HL, HL, seed=parallel.image_seed(1234, i))
    return ctx.sample_image(c, unc, 7.5, STEPS, init_latent=lat)[0]


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist

    from stable_diffusion_burn_b200 import _lib, parallel
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        ctx = _lib.Context(rank)
        if rank == 0:
            ctx.init_synthetic(0)
        parallel.broadcast_weights(ctx, rank, world)  # ranks > 0 start from a zeroed arena: everything they know comes from here
        ctx.finalize_weights()
        idx = parallel.shard_images(N_IMAGES, rank, world)
        imgs = np.stack([_sample(ctx, i) for i in idx])
        full = parallel.gather_images(imgs, N_IMAGES, rank, world)  # NCCL gather of device buffers
        # the broadcast really shipped the weights: one tensor read back on every rank
        w = ctx.get_tensor("unet/input_blocks/rt1/res/conv_in/weight", (320, 320, 3, 3))
        q.put((rank, None if full is None else full, float(np.abs(w).sum())))
        ctx.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
def test_world2_images_bit_identical_to_world1(ctx):
    import torch.multiprocessing as mp
    ctx.init_synthetic(0)
    ctx.finalize_weights()
    want = np.stack([_sample(ctx, i) for i in range(N_IMAGES)])  # world 1: every image on this process' GPU 0 context
    wsum = float(np.abs(ctx.get_tensor("unet/input_blocks/rt1/res/conv_in/weight", (320, 320, 3, 3))).sum())
    mpc = mp.get_context("spawn")
    q = mpc.Queue()
    port = _free_port()
    procs = [mpc.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    full = [r[1] for r in res if r[1] is not None][0]
    assert all(abs(r[2] - wsum) == 0.0 for r in res), "weights differ between ranks after the broadcast"
    assert full.shape == want.shape
    assert np.array_equal(full, want), "an image depends on the rank count"

"""Every rank of the data-parallel Trainer.train must see the same global batches (each then trains its own chunk).  The
reference's data order comes from host generators that each process seeds from OS entropy: BucketingSampler shuffles
the ids inside every bin and, under --shuffle, the bins themselves with np.random (utils/data_loader.py), and
SpectrogramDataset picks a manifest with random.randint; the DataLoader draws its workers' base seed from torch's CPU
generator.  parallel.seed_host_rngs, which the data-parallel loop calls at its start, seeds all three from rank 0.

Two gloo ranks on the CPU, seeded differently, drive the reference's own BucketingSampler over a duration-sorted dataset
with many equal lengths (which _collate_fn's stable sort keeps in sampler order) through two shuffled epochs, with 0 and
2 loader workers: with seed_host_rngs they see identical global batches, without it they do not."""
import importlib
import os
import random
import socket
import sys
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ref_shim

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")

LENGTHS = [12] * 7 + [10] * 9 + [9] * 5 + [7] * 11          # a manifest sorted by duration: many ties


class Utterances(torch.utils.data.Dataset):
    """(frames, id, manifest) per index; the manifest is picked as SpectrogramDataset.__getitem__ picks it."""

    def __len__(self):
        return len(LENGTHS)

    def __getitem__(self, i):
        return LENGTHS[i], i, random.randint(0, 2)


def collate(batch):
    """_collate_fn's order: longest first, stable among equal lengths."""
    return [(i, m) for _, i, m in sorted(batch, key=lambda x: x[0], reverse=True)]


def _reference_sampler():
    import scipy.signal
    for name in ("librosa", "torchaudio"):                  # imported by utils/data_loader.py, not used by the sampler
        try:
            importlib.import_module(name)
        except ImportError:
            sys.modules[name] = types.ModuleType(name)
    for name in ("hamming", "hann", "blackman", "bartlett"):    # scipy >= 1.13 keeps them in scipy.signal.windows only
        if not hasattr(scipy.signal, name):
            setattr(scipy.signal, name, getattr(scipy.signal.windows, name))
    Sampler = torch.utils.data.Sampler
    if Sampler.__init__ is object.__init__:                  # torch >= 2.2 dropped Sampler(data_source), which it calls
        Sampler.__init__ = lambda self, data_source=None: None
    ref_shim.load([])
    return importlib.import_module("utils.data_loader").BucketingSampler


def _worker(rank, world, port, seeded, workers, q):
    import b200asr
    parallel = importlib.import_module(b200asr.__name__ + ".parallel")
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    random.seed(1000 + rank)                                 # stands in for each process's own OS-entropy seed
    np.random.seed(2000 + rank)
    torch.manual_seed(3000 + rank)
    BucketingSampler = _reference_sampler()
    if seeded:
        parallel.seed_host_rngs()
    data = Utterances()
    sampler = BucketingSampler(data, batch_size=4)
    loader = torch.utils.data.DataLoader(data, batch_sampler=sampler, num_workers=workers, collate_fn=collate)
    seen = []
    for epoch in range(2):
        seen += [b for b in loader]
        sampler.shuffle(epoch)                               # trainer.py:210-213 under --shuffle
    q.put((rank, seen))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("seeded", [True, False])
def test_ranks_see_the_same_global_batches(seeded, workers):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, seeded, workers, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=120)
    assert [p.exitcode for p in procs] == [0, 0]
    got = dict(q.get(timeout=10) for _ in range(2))
    a, b = got[0], got[1]
    assert len(a) == len(b) == 2 * ((len(LENGTHS) + 3) // 4)
    for epoch in (a[:len(a) // 2], a[len(a) // 2:]):         # every epoch visits each utterance once
        assert sorted(i for batch in epoch for i, _ in batch) == list(range(len(LENGTHS)))
    if seeded:
        assert a == b
    else:
        assert a != b                                        # what the ranks would train on without the common seed

"""GPU: ops.png_decode_gray8 bit-identical to cv2.imdecode(..., IMREAD_GRAYSCALE) on the recordings' maps, on cv2-encoded images of
every compression level and strategy, on streams built here with zlib (every row filter, stored and fixed-Huffman blocks), in a
large permuted batch; malformed streams flagged with every other byte untouched; and both training loaders against the host
decoder."""
import shutil
import zlib

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from lav_b200 import data_paint, ops, png, synth  # noqa: E402
from lav_b200.capi import LavbError  # noqa: E402
from tests.test_gpu_bev_train import bev_config, gold_ds  # noqa: E402,F401
from tests.test_gpu_temporal_dataset import config, gold  # noqa: E402,F401
from tests.test_png_host_cpu import chunk, split_chunks  # noqa: E402

pytestmark = pytest.mark.gpu
CANARY = 0xAB


def decode(streams, h, w, cuda, order=None):
    """streams -> (planes (n, h, w) numpy, status numpy, canaries intact); job k writes plane 2 * order[k] + 1 of a buffer of
    0xAB planes, so every plane has an untouched canary plane on both sides."""
    n = len(streams)
    order = np.arange(n) if order is None else np.asarray(order)
    jobs = np.zeros(n, ops.PNG_JOB_DTYPE)
    lens = np.array([len(s) for s in streams], np.int64)
    jobs["off"], jobs["len"], jobs["dst"], jobs["h"], jobs["w"] = np.cumsum(lens) - lens, lens, 2 * order + 1, h, w
    src = torch.from_numpy(np.frombuffer(b"".join(streams) or b"\0", np.uint8).copy()).to(cuda)
    out = torch.full((2 * n + 1, h, w), CANARY, dtype=torch.uint8, device=cuda)
    status = ops.png_decode_gray8(src, jobs, out)
    out = out.cpu().numpy()
    return out[2 * order + 1], status.cpu().numpy(), bool((out[0::2] == CANARY).all())


def cv2_decode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_GRAYSCALE)


def test_every_map_of_a_recording(cuda, tmp_path):
    paths = synth.record_trajectories(str(tmp_path), 2, 24, seed=11)
    datas = [data_paint.open_env(p).get(f"map_{c}_{i:05d}") for p in paths for i in range(24) for c in range(12)]
    streams = [png.parse(d, "k", 320)[0] for d in datas]
    planes, status, canary = decode(streams, 320, 320, cuda)
    assert canary and not status.any()
    for d, got in zip(datas, planes):
        assert np.array_equal(got, cv2_decode(d))


def images(h, w, rs):
    yield (rs.rand(h, w) > 0.8).astype(np.uint8) * 255
    yield rs.randint(0, 256, (h, w), dtype=np.uint8)
    yield (np.add.outer(np.arange(h) * 3, np.arange(w)) % 256).astype(np.uint8)
    yield np.full((h, w), 77, np.uint8)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 320), (320, 1), (7, 13), (320, 320), (1024, 1024)])
def test_cv2_encoded_images_every_level_and_strategy(cuda, h, w):
    rs = np.random.RandomState(h * 7 + w)
    datas = [cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, lvl, cv2.IMWRITE_PNG_STRATEGY, strat])[1].tobytes()
             for img in images(h, w, rs) for lvl in range(10) for strat in range(5)]
    streams = [png.chunks(d, "k")[1] for d in datas]
    planes, status, canary = decode(streams, h, w, cuda, rs.permutation(len(streams)))
    assert canary and not status.any(), np.nonzero(status)
    for k, (d, got) in enumerate(zip(datas, planes)):
        assert np.array_equal(got, cv2_decode(d)), k


def filter_rows(img, types):
    """the PNG row filters of an (h, w) uint8 image, row r with filter types[r] -> the filtered scanlines."""
    h, w = img.shape
    x = img.astype(np.int32)
    out = []
    for r in range(h):
        cur, prv = x[r], (x[r - 1] if r else np.zeros(w, np.int32))
        a, b, c = np.concatenate([[0], cur[:-1]]), prv, np.concatenate([[0], prv[:-1]])
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        pred = [0, a, b, (a + b) // 2, np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))][types[r]]
        out.append(bytes([types[r]]) + ((cur - pred) % 256).astype(np.uint8).tobytes())
    return b"".join(out)


def fixed_huffman(raw):
    c = zlib.compressobj(9, zlib.DEFLATED, 15, 9, zlib.Z_FIXED)
    return c.compress(raw) + c.flush()


@pytest.mark.parametrize("encode", ["stored", "fixed", "dynamic"])
def test_every_row_filter(cuda, encode):
    rs = np.random.RandomState(3)
    enc = {"stored": lambda r: zlib.compress(r, 0), "fixed": fixed_huffman, "dynamic": lambda r: zlib.compress(r, 6)}[encode]
    for h, w in [(1, 1), (7, 13), (64, 80), (320, 320)]:
        imgs = [rs.randint(0, 256, (h, w), dtype=np.uint8), (rs.rand(h, w) > 0.7).astype(np.uint8) * 255]
        types = [[f] * h for f in range(5)] + [list(rs.randint(0, 5, h))]
        cases = [(img, t) for img in imgs for t in types]
        planes, status, canary = decode([enc(filter_rows(img, t)) for img, t in cases], h, w, cuda)
        assert canary and not status.any()
        for k, ((img, _), got) in enumerate(zip(cases, planes)):
            assert np.array_equal(got, img), (h, w, k)


def test_mixed_batch_of_2304_permuted(cuda):
    rs = np.random.RandomState(9)
    datas = []
    for k in range(2304):
        img = (rs.rand(320, 320) > rs.uniform(0.5, 0.99)).astype(np.uint8) * 255 if k % 3 else rs.randint(0, 256, (320, 320), np.uint8)
        datas.append(cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, int(k % 10)])[1].tobytes())
    planes, status, canary = decode([png.parse(d, "k", 320)[0] for d in datas], 320, 320, cuda, rs.permutation(2304))
    assert canary and not status.any()
    for d, got in zip(datas, planes):
        assert np.array_equal(got, cv2_decode(d))


def bitstream(fields):
    """LSB-first packing of (value, n bits) fields, with 8 zero bytes after (so only the error under test can stop a decoder)."""
    v, n = 0, 0
    for val, nb in fields:
        v |= val << n
        n += nb
    return v.to_bytes((n + 7) // 8 + 8, "little")


def malformed(raw, good):
    return {
        "truncated": good[:-12],
        "adler": good[:-1] + bytes([good[-1] ^ 1]),
        "block_type_3": b"\x78\x01" + bitstream([(1, 1), (3, 2)]),
        "len_nlen": b"\x78\x01" + bytes([1, 5, 0, 0xFB, 0xFE]) + b"hello" + b"\0" * 8,
        # fixed block opening with a match (length code 257, 7 bits 0000001 sent MSB first, distance code 0): distance 1 > 0 bytes
        "distance_before_start": b"\x78\x01" + bitstream([(1, 1), (1, 2)] + [(0, 1)] * 6 + [(1, 1)] + [(0, 5)]),
        # dynamic block whose code-length code has three 1-bit codes
        "oversubscribed": b"\x78\x01" + bitstream([(1, 1), (2, 2), (0, 5), (0, 5), (15, 4)] + [(1, 3)] * 3 + [(0, 3)] * 16),
        "filter_5": zlib.compress(b"\x05" + raw[1:], 1),
        "short": zlib.compress(raw[:-7], 1),
        "long": zlib.compress(raw + b"\0", 1),
        "header": b"\x78\x02" + good[2:],
        "dictionary": b"\x78\x20" + good[2:],
        "empty": b"",
    }


def test_malformed_streams_are_flagged_and_contained(cuda):
    rs = np.random.RandomState(2)
    imgs = [(rs.rand(320, 320) > 0.8).astype(np.uint8) * 255 for _ in range(3)]
    raws = [filter_rows(i, [1] * 320) for i in imgs]
    goods = [zlib.compress(r, 1) for r in raws]
    for name, bad in malformed(raws[1], goods[1]).items():
        planes, status, canary = decode([goods[0], bad, goods[2]], 320, 320, cuda)
        assert canary, name
        assert status[1] != 0 and status[0] == 0 and status[2] == 0, (name, status)
        assert np.array_equal(planes[0], imgs[0]) and np.array_equal(planes[2], imgs[2]), name


def test_bad_arguments_rejected_before_launch(cuda):
    good = zlib.compress(filter_rows(np.zeros((8, 8), np.uint8), [0] * 8))
    src = torch.from_numpy(np.frombuffer(good, np.uint8).copy()).to(cuda)
    out = torch.full((2, 8, 8), CANARY, dtype=torch.uint8, device=cuda)
    job = np.zeros(1, ops.PNG_JOB_DTYPE)
    job["len"], job["dst"], job["h"], job["w"] = len(good), 1, 8, 8

    def variant(**kw):
        j = job.copy()
        for k, v in kw.items():
            j[k] = v
        return j
    bad = [(src, variant(dst=2), out), (src, variant(dst=-1), out), (src, variant(h=9), out), (src, variant(w=7), out),
           (src, variant(len=len(good) + 1), out), (src, variant(off=-1), out), (src, np.concatenate([job, job]), out),
           (src.cpu(), job, out), (src, job, out.cpu()), (src.to(torch.int32), job, out), (src, job, out[:, :, :4]),
           (src, job, out.view(16, 8)), (src, job, out.float())]
    for s, j, o in bad:
        with pytest.raises(LavbError):
            ops.png_decode_gray8(s, j, o)
    with pytest.raises(LavbError):
        ops.png_decode_gray8(src, job, out, status=torch.zeros(2, dtype=torch.int32, device=cuda))
    torch.cuda.synchronize()
    assert (out == CANARY).all()
    assert ops.png_decode_gray8(src, job, out).cpu().tolist() == [0] and (out[1] == 0).all() and (out[0] == CANARY).all()


def host_bev(ds, hs, trajs):
    """the BEV targets of the prepared samples ``hs`` (of trajectories ``trajs``) from map planes decoded by synth.decode_png."""
    from lav_b200.datasets import bev_job_table
    planes = [synth.decode_png(ds.env(t).get(key.rsplit(": ", 1)[-1])) for h, t in zip(hs, trajs) for key, _ in h["pngs"]]
    n_bev = 3 + 2 * (ds.num_frame_stack + 1)
    out = torch.empty((len(hs), n_bev, 320, 320), dtype=torch.uint8, device=ds.device)
    return ops.bev_targets(torch.from_numpy(np.stack(planes)).to(ds.device), bev_job_table(hs, n_bev), out)


@pytest.mark.parametrize("num_workers,rank", [(1, 0), (8, 0), (8, 1)])
def test_lidar_loader_and_samples_equal_host_decode(cuda, gold, config, num_workers, rank):  # noqa: F811
    from lav_b200.datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
    ds = TemporalLiDARPaintedDataset(config, seed=int(gold["seed"]), device=cuda)
    loader = TemporalBatchLoader(ds, 2, seed=5, rank=rank, world=2, num_workers=num_workers)
    got = list(loader)
    rng, gen = loader.generators(0)
    order = loader.shard(0)
    for k, batch in enumerate(got):
        idxs = order[k * loader.B:(k + 1) * loader.B]
        draws = [ds.draw(rng) for _ in idxs]
        hs = [ds.prepare(int(i), *d) for i, d in zip(idxs, draws)]
        want = host_bev(ds, hs, [ds.index[int(i)][0] for i in idxs])
        assert torch.equal(batch[5], want), k
        assert torch.equal(ds.sample_batch(idxs, draws, torch.Generator().manual_seed(k))[5], want), k
        for b, (i, d) in enumerate(zip(idxs, draws)):
            assert torch.equal(ds.sample(int(i), *d)[5], want[b]), (k, b)


@pytest.mark.parametrize("num_workers,rank", [(1, 0), (8, 0), (8, 1)])
def test_bev_loader_and_samples_equal_host_decode(cuda, gold_ds, bev_config, num_workers, rank):  # noqa: F811
    from lav_b200.datasets import TemporalBEVBatchLoader, TemporalBEVDataset
    ds = TemporalBEVDataset(bev_config, seed=int(gold_ds["seed"]), device=cuda)
    loader = TemporalBEVBatchLoader(ds, 2, seed=5, rank=rank, world=2, num_workers=num_workers)
    got = list(loader)
    assert len(got) == len(loader) >= 1
    gen = torch.Generator(device="cpu").manual_seed(5 * 1000003 + 0 * 1009 + rank)
    order = loader.shard(0)
    for k, batch in enumerate(got):
        idxs = order[k * loader.B:(k + 1) * loader.B]
        draws = [ds.draw(gen) for _ in idxs]
        hs = [ds.prepare(int(i), *d) for i, d in zip(idxs, draws)]
        want = host_bev(ds, hs, [ds.index[int(i)][0] for i in idxs])
        assert torch.equal(batch[0], want), k
        for b, (i, d) in enumerate(zip(idxs, draws)):
            assert torch.equal(ds.sample(int(i), *d)[0], want[b]), (k, b)


def corrupt_adler(data):
    """a PNG with valid chunks whose zlib stream has a wrong Adler-32."""
    parts = split_chunks(data)
    stream = b"".join(b for t, b in parts if t == b"IDAT")
    stream = stream[:-1] + bytes([stream[-1] ^ 0x10])
    return png.SIGNATURE + chunk(b"IHDR", parts[0][1]) + chunk(b"IDAT", stream) + chunk(b"IEND", b"")


@pytest.mark.parametrize("which", ["lidar", "bev"])
def test_a_corrupted_map_raises_before_its_batch(cuda, gold, config, gold_ds, bev_config, which, tmp_path):  # noqa: F811
    import yaml
    from lav_b200.datasets import (TemporalBatchLoader, TemporalBEVBatchLoader, TemporalBEVDataset,
                                   TemporalLiDARPaintedDataset)
    src_cfg = config if which == "lidar" else bev_config
    cfg = yaml.safe_load(open(src_cfg))
    shutil.copytree(cfg["data_dir"], tmp_path / "data")
    cfg["data_dir"] = str(tmp_path / "data")
    yaml.safe_dump(cfg, open(tmp_path / "c.yaml", "w"))
    Ds, Loader = ((TemporalLiDARPaintedDataset, TemporalBatchLoader) if which == "lidar" else
                  (TemporalBEVDataset, TemporalBEVBatchLoader))
    ds = Ds(str(tmp_path / "c.yaml"), seed=1, device=cuda)
    loader = Loader(ds, 2, seed=5, num_workers=2)
    first = loader.shard(0)[0]
    traj, index = ds.index[int(first)]
    key = f"map_0_{index:05d}"
    env = data_paint.open_env(ds.paths[traj], write=True)
    env.put(key, corrupt_adler(env.get(key)))
    env.close()
    got = []
    with pytest.raises(LavbError, match=key):
        for batch in loader:
            got.append(batch)
    assert not got

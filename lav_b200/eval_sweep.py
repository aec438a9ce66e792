"""Checkpoint sweeps and multi-rank runs of the evaluators (lav_b200.evaluate, lav_b200.evaluate_bev).

Sweeps.  K checkpoints are scored in one pass over a recording: each batch is loaded and staged once, then every checkpoint runs
its own models and scoring launches on it into its own host accumulators.  All K checkpoints stay resident on the device;
check_sweep_fits refuses a sweep that would not fit before any data is loaded.

Ranks.  Under torchrun every rank scores the contiguous sample range [r * n // N, (r + 1) * n // N) (TemporalBatchLoader's
ordered shard).  gather_merged gathers the ranks' host accumulators to rank 0 over a gloo group and folds them in rank order,
which is sample-index order: every accumulator's ``extend`` sums its integer counts and appends its per-sample records, so rank 0's
summary() sees exactly the records one process would have collected.  Any object with an ``extend`` method can be merged.

Checkpoint selection for the CLIs: several weight paths paired by position, or --run-dir [--epochs] finding the {name}_{epoch}.th
files train_full / train_bev write.
"""
import os
import re

import torch
import torch.distributed as dist

from .capi import LavbError

# device memory an evaluation needs besides its resident checkpoints, per sample of a batch: the batch itself and the activations
# of one checkpoint's forward and scoring; DESIGN §4 measures about 70 MB per sample (2.24 GB at B = 32 with --forecast
# --plan-safety, 30 000-point sweeps, H100), and this keeps a margin above it
EVAL_WORKSPACE_BYTES_PER_SAMPLE = 96 << 20


# ---------------------------------------------------------------------------------------------------- ranks
def rank_and_world():
    """(rank, world size) of the default process group, (0, 1) without one."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def eval_device():
    """the device of this rank: cuda:(LOCAL_RANK % device_count), so several ranks may share a GPU."""
    return torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)) % torch.cuda.device_count())


def init_ranks():
    """under torchrun (WORLD_SIZE > 1) a gloo process group for the host-side merge; -> True when one was created here."""
    if int(os.environ.get("WORLD_SIZE", 1)) > 1 and not dist.is_initialized():
        dist.init_process_group("gloo")
        return True
    return False


def merge_ranks(parts):
    """fold the per-rank accumulator structures ``parts`` (a list in rank order of equal nests of lists / tuples / dicts whose
    leaves have ``extend``) into the first one, in rank order.  -> the merged structure."""
    def fold(a, b):
        if isinstance(a, dict):
            for k in a:
                fold(a[k], b[k])
        elif isinstance(a, (list, tuple)):
            if len(a) != len(b):
                raise LavbError(f"ranks hold {len(a)} and {len(b)} accumulators")
            for x, y in zip(a, b):
                fold(x, y)
        else:
            a.extend(b)
    merged = parts[0]
    for p in parts[1:]:
        fold(merged, p)
    return merged


def gather_merged(accumulators):
    """the accumulators of every rank gathered to rank 0 over gloo and merged in rank order (merge_ranks); None on the other
    ranks.  Without a process group, or with one rank, ``accumulators`` itself."""
    rank, world = rank_and_world()
    if world == 1:
        return accumulators
    group = None if dist.get_backend() == "gloo" else dist.new_group(backend="gloo")
    parts = [None] * world if rank == 0 else None
    dist.gather_object(accumulators, parts, dst=0, group=group)
    return merge_ranks(parts) if rank == 0 else None


# ---------------------------------------------------------------------------------------------------- device memory
def module_tensors(*modules):
    """the distinct parameter and buffer tensors of ``modules``."""
    seen = {}
    for m in modules:
        for t in list(m.parameters()) + list(m.buffers()):
            seen[id(t)] = t
    return list(seen.values())


class ResidentMeter:
    """the device bytes the first checkpoint of a sweep takes: what the allocator gained while it was moved and packed, plus
    its tensors that were already on the device."""

    def __init__(self, device, *modules):
        self.device = device = torch.device("cuda", torch.device(device).index if torch.device(device).index is not None
                                            else torch.cuda.current_device())
        torch.cuda.synchronize(device)
        free, _ = torch.cuda.mem_get_info(device)
        self.allocated = torch.cuda.memory_allocated(device)
        self.already = sum(t.numel() * t.element_size() for t in module_tensors(*modules) if t.device == device)
        # what this process could hold: the free memory, its cache's slack and the checkpoint's own tensors
        self.available = free + torch.cuda.memory_reserved(device) - self.allocated + self.already

    def resident(self):
        torch.cuda.synchronize(self.device)
        return torch.cuda.memory_allocated(self.device) - self.allocated + self.already


def sweep_capacity(per_checkpoint, available, workspace):
    """the largest number of checkpoints of ``per_checkpoint`` bytes that fit in ``available`` bytes beside ``workspace``."""
    return max(0, (available - workspace) // max(1, per_checkpoint))


def check_sweep_fits(k, per_checkpoint, available, batch_size, what="checkpoints"):
    """refuse a sweep of ``k`` resident checkpoints that would not fit (a single checkpoint is never refused)."""
    workspace = EVAL_WORKSPACE_BYTES_PER_SAMPLE * batch_size
    cap = sweep_capacity(per_checkpoint, available, workspace)
    if k > 1 and k > cap:
        raise LavbError(f"a sweep of {k} {what} does not fit on the device: each takes {per_checkpoint / 2**20:.1f} MiB resident, "
                        f"{available / 2**30:.1f} GiB are available and a batch of {batch_size} needs {workspace / 2**30:.1f} GiB "
                        f"besides; at most {cap} fit")
    return cap


# ---------------------------------------------------------------------------------------------------- checkpoint selection
def parse_epochs(spec):
    """"1,8,16-64" -> the sorted distinct epochs."""
    out = set()
    for part in spec.split(","):
        part = part.strip()
        m = re.fullmatch(r"(\d+)(?:-(\d+))?", part)
        if not m:
            raise LavbError(f"--epochs: {part!r} is neither an epoch nor a range a-b")
        a, b = int(m.group(1)), int(m.group(2) or m.group(1))
        if b < a:
            raise LavbError(f"--epochs: the range {part} is empty")
        out.update(range(a, b + 1))
    return sorted(out)


def find_checkpoints(run_dir, names, epochs=None):
    """the checkpoints {name}_{epoch}.th in ``run_dir``, one per epoch, each with a file for every entry of ``names``, sorted by
    epoch; only ``epochs`` when given.  -> [(epoch, {name: path})].  An epoch with some of its files missing, and an empty
    selection, are refused with the missing file named."""
    if not os.path.isdir(run_dir):
        raise LavbError(f"--run-dir {run_dir} is not a directory")
    found = {}
    for f in os.listdir(run_dir):
        m = re.fullmatch(r"(\w+?)_(\d+)\.th", f)
        if m and m.group(1) in names:
            found.setdefault(int(m.group(2)), set()).add(m.group(1))
    wanted = sorted(found) if epochs is None else epochs
    if not wanted:
        raise LavbError(f"no {' / '.join(n + '_{epoch}.th' for n in names)} checkpoint in {run_dir}")
    out = []
    for e in wanted:
        paths = {n: os.path.join(run_dir, f"{n}_{e}.th") for n in names}
        for n in names:
            if n not in found.get(e, ()):
                raise LavbError(f"epoch {e}: {paths[n]} is missing")
        out.append((e, paths))
    return out


def pair_paths(named_lists):
    """{name: [paths]} given on the command line, paired by position -> [(None, {name: path})]; unequal counts are refused with
    the unpaired paths named."""
    counts = {n: len(p) for n, p in named_lists.items()}
    if len(set(counts.values())) != 1:
        k = min(counts.values())
        extra = [p for ps in named_lists.values() for p in ps[k:]]
        raise LavbError(f"the weight lists pair by position but their lengths differ ({counts}): {', '.join(extra)} "
                        f"{'has' if len(extra) == 1 else 'have'} no partner")
    names = list(named_lists)
    return [(None, {n: named_lists[n][i] for n in names}) for i in range(counts[names[0]])]


def select_checkpoints(args, names):
    """the checkpoints of parsed CLI arguments: --run-dir [--epochs], or the --{name}-weights lists paired by position."""
    lists = {n: getattr(args, f"{n}_weights") for n in names}
    if args.run_dir is not None:
        if any(lists.values()):
            raise LavbError("give either --run-dir or weight paths, not both")
        return find_checkpoints(args.run_dir, names, parse_epochs(args.epochs) if args.epochs else None)
    if args.epochs:
        raise LavbError("--epochs selects checkpoints of --run-dir")
    missing = [f"--{n}-weights" for n, p in lists.items() if not p]
    if missing:
        raise LavbError(f"{' and '.join(missing)} or --run-dir is required")
    return pair_paths(lists)


def add_checkpoint_args(ap, names, help_of):
    """the checkpoint options of an evaluator's CLI for the files ``names``."""
    for n in names:
        ap.add_argument(f"--{n}-weights", nargs="+", default=None, help=help_of[n] + "; several paths make a sweep, paired by position")
    ap.add_argument("--run-dir", default=None,
                    help=f"score the {' / '.join(n + '_{epoch}.th' for n in names)} checkpoints of a training run in this directory")
    ap.add_argument("--epochs", default=None, help="with --run-dir: the epochs to score, e.g. 1,8,16-64 (default: every one found)")


# ---------------------------------------------------------------------------------------------------- reports
def sweep_json(checkpoints, results, samples, world):
    """the --json document of a sweep of K > 1 checkpoints."""
    return dict(samples=samples, ranks=world,
                checkpoints=[dict(epoch=e, weights=w, result=r) for (e, w), r in zip(checkpoints, results)])


def sweep_table(checkpoints, rows):
    """one line per checkpoint: its epoch (or its first path) and the (column, value) pairs of ``rows``."""
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    labels = [f"epoch {e}" if e is not None else next(iter(w.values())) for e, w in checkpoints]
    width = max(len(s) for s in labels)
    head = [c for c, _ in rows[0]]
    cells = [[fmt(v) for _, v in r] for r in rows]
    widths = [max(len(h), *(len(c[i]) for c in cells)) for i, h in enumerate(head)]
    line = lambda first, cols: "  ".join([first.ljust(width)] + [c.rjust(w) for c, w in zip(cols, widths)])
    return "\n".join([line("checkpoint", head)] + [line(s, c) for s, c in zip(labels, cells)])

"""Frame pipeline: the GPU side of LAVAgent.run_step (team_code_v2/lav_agent_fast.py:205-360) for B
independent agent ticks at once — seg -> paint -> sweep stack -> LiDAR model -> detection decode ->
UniPlanner -> brake.  The CARLA shell (sensors, EKF, PID, route commands) stays where it is; it hands
this class the tensors it already holds and gets back what it feeds to the PID / safety logic.

State per agent (``SweepHistory``): the FIFO of painted sweeps + ego poses that get_stacked_lidar reads
(lav_agent_fast.py:363-383), resident on the device.
"""
import contextlib
import copy
import math
from collections import deque

import os

import numpy as np
import torch

from . import ops
from .model_inference import InferModel

FUSE_SEG_HEAD = True  # ERFNet's last layer (ConvTranspose2d 16->5, k2 s2) + softmax evaluated inside the painting gather
FORK_BRAKE = True     # run the brake predictor as a parallel branch of the perception graph
STEM_U8 = True        # brake-model stem (7x7 s2 on 3 channels) in the lav_b200 kernel, straight from the camera bytes
NUM_REPEAT = 4
GAP = NUM_REPEAT + 1          # lav_agent_fast.py:31-32
NUM_FRAME_STACK = 2           # team_code_v2/config.yaml: num_frame_stack
MAX_LIDAR_POINTS = 120000


class SweepHistory:
    """FIFO of fused sweeps (N,8) with the ego pose they were taken at (lav_agent_fast.py:267-274)."""

    def __init__(self, num_frame_keep=(NUM_FRAME_STACK + 1) * GAP):
        self.lidars, self.locs, self.oris = deque(), deque(), deque()
        self.keep = num_frame_keep

    def push(self, fused, loc, ori):
        self.lidars.append(fused)
        self.locs.append(np.asarray(loc, dtype=np.float64))
        self.oris.append(float(ori))
        if len(self.lidars) > self.keep:
            self.lidars.popleft(); self.locs.popleft(); self.oris.popleft()

    def selected(self):
        """sweeps get_stacked_lidar picks: t, t-GAP, t-2*GAP ... (newest first)."""
        idx = list(range(len(self.lidars) - 1, -1, -GAP))[:NUM_FRAME_STACK + 1]
        return [(self.lidars[t], self.locs[t], self.oris[t]) for t in idx]


def stack_into(dst, sweeps, roof_filter=False):
    """get_stacked_lidar + move_lidar_points (lav_agent_fast.py:363-383,547-565) into rows of dst (P,11).
    sweeps: [(fused (n,8), loc, ori)] newest first.  Returns the number of rows written."""
    loc0, ori0 = sweeps[0][1], sweeps[0][2]
    c0, s0 = math.cos(ori0), math.sin(ori0)
    row = 0
    for i, (s, loc, ori) in enumerate(sweeps):
        d = ori - ori0
        R = np.array([[math.cos(d), math.sin(d), 0], [-math.sin(d), math.cos(d), 0], [0, 0, 1]])
        dl = (loc - loc0) @ np.array([[c0, -s0], [s0, c0]])
        n = s.shape[0]
        ops.stack_sweep(s, R, dl[0], dl[1], i, NUM_FRAME_STACK + 1, dst[row:row + n], roof_filter=roof_filter)
        row += n
    return row


def infer_model(lidar_model, uniplanner, precision, camera_x, camera_z, device):
    """The InferModel of the agent at ``precision``: ``lidar_model`` switched to it in place; the UniPlanner's embedder cast on a
    PRIVATE copy of ``uniplanner``, so a model object shared with a trainer / checkpoint writer / fp32 parity check keeps its fp32
    master weights."""
    lidar_model.set_precision(precision)
    dt = ops.h16() if precision == "f16" else torch.float32
    up = copy.deepcopy(uniplanner)
    up.lidar_conv_emb.to(dt).to(memory_format=torch.channels_last)
    return InferModel(lidar_model, up, camera_x, camera_z, device)


def brake_model(bra_model, precision):
    """The brake model the agent runs at ``precision``: a PRIVATE copy of ``bra_model`` (so a model object shared with a trainer /
    checkpoint writer keeps its fp32 master weights) with its trunk and attention pools cast to the 16-bit type for "f16"."""
    dt = ops.h16() if precision == "f16" else torch.float32
    bra = copy.deepcopy(bra_model)
    bra.conv_backbone.to(dt).to(memory_format=torch.channels_last)
    bra.attn1.to(dt); bra.attn2.to(dt)
    return bra


def brake_probs(bra, rgbs_u8, tel_u8, u8=True):
    """pred_bra (B,) of a brake_model copy on the camera bytes: rgbs_u8 (B, 3, H, W, 3) the three cameras side by side, tel_u8
    (B, h, w, 3).  A 16-bit copy runs forward_u8 (the stem kernel on the raw bytes) when ``u8`` and STEM_U8; otherwise the float
    call of lav_agent_fast.py:257-262,318-321 on the stitched wide view, which the caller runs under math_mode(precision)."""
    if u8 and STEM_U8 and bra.conv_backbone.conv1.weight.dtype == ops.h16():
        return bra.forward_u8(rgbs_u8, tel_u8)
    B, n, H, W, _ = rgbs_u8.shape
    wide = rgbs_u8.permute(0, 2, 1, 3, 4).reshape(B, H, n * W, 3).permute(0, 3, 1, 2).float()
    tel = tel_u8.permute(0, 3, 1, 2).float()
    return bra(wide.contiguous(memory_format=torch.channels_last), tel.contiguous(memory_format=torch.channels_last))


@contextlib.contextmanager
def math_mode(precision):
    """exact path: the cuDNN / cuBLAS heads must not drop to TF32 — scoped to the caller's block, the process-wide flags are
    restored afterwards."""
    if precision != "fp32":
        yield
        return
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


class FramePipeline:
    def __init__(self, seg_model, lidar_model, uniplanner, bra_model, camera_x=1.5, camera_z=2.4, device=torch.device("cuda"),
                 precision="f16"):
        self.device = device
        self.seg_model = seg_model.to(device).eval()
        # the PyTorch heads are cast for the 16-bit path: the pipeline works on PRIVATE copies, so a model object shared with a
        # trainer / checkpoint writer / fp32 parity check keeps its fp32 master weights (set_precision re-copies from these)
        self._src_uniplanner = uniplanner.to(device).eval()
        self._src_bra = bra_model.to(device).eval() if bra_model is not None else None
        self._lidar_model, self._cam = lidar_model.to(device).eval(), (camera_x, camera_z)
        self.bra_model = None
        self.set_precision(precision)

    def set_precision(self, precision):
        assert precision in ("fp32", "f16"), precision
        self.precision = precision
        self.seg_model.set_precision(precision)
        self.infer_model = infer_model(self._lidar_model, self._src_uniplanner, precision, self._cam[0], self._cam[1], self.device)
        if self._src_bra is not None:
            self.bra_model = brake_model(self._src_bra, precision)
        return self

    def _math_mode(self):
        return math_mode(self.precision)

    @torch.no_grad()
    def step(self, rgbs_u8, tel_u8, lidars, histories, nxps, cmds, poses=None):
        with self._math_mode():
            return self._step(rgbs_u8, tel_u8, lidars, histories, nxps, cmds, poses)

    def _step(self, rgbs_u8, tel_u8, lidars, histories, nxps, cmds, poses=None):
        """One tick of B agents.
        rgbs_u8 (B,3,288,256,3) uint8 RGB; tel_u8 (B,192,480,3) uint8 or None; lidars: list of (N_b,4) fp32 (roof-filtered
        current sweep, lav_agent_fast.py:233-247); histories: list of SweepHistory (updated in place); nxps (B,2); cmds (B,)
        poses: list of (loc, ori) of this tick (EKF state); default = zero motion.
        Returns dict(ego_plan_locs (B,20,2), ego_cast_locs, other_cast_locs [B], other_cast_cmds [B], pred_bra (B,), det, pred_bev)."""
        B = rgbs_u8.shape[0]
        im = self.infer_model
        # (1) semantic segmentation of the 3 cameras of every agent: logits NHWC (B*3,288,256,5)
        imgs = rgbs_u8.reshape(B * 3, *rgbs_u8.shape[2:])
        if FUSE_SEG_HEAD:
            feat, table, ncls = self.seg_model.forward_features_nhwc(imgs)
            cams = np.stack([c.packed() for c in im.coord_converters])
        else:
            logits = self.seg_model.forward_nhwc(imgs)
            logits = logits.view(B, 3, *logits.shape[1:]).permute(0, 1, 4, 2, 3)      # logical (B,3,5,H,W), channels-last storage
        # (2) paint the current sweep (softmax + background suppression fused into the gather) and push to the FIFO
        for b in range(B):
            if FUSE_SEG_HEAD and table is not None:
                cur = lidars[b].float().contiguous()[None]
                fused = ops.paint_deconv_batched(cur, feat[3 * b:3 * b + 3], ncls, table, cams, cur.shape[2],
                                                 torch.empty((1, cur.shape[1], cur.shape[2] + ncls - 1), device=self.device),
                                                 tuple(rgbs_u8.shape[2:4]))[0]
            else:
                if FUSE_SEG_HEAD:
                    raise RuntimeError("FUSE_SEG_HEAD needs the v2 output_conv (ConvTranspose2d 16->C, k2 s2)")
                fused = im.forward_paint(lidars[b], logits[b], logits=True)
            loc, ori = poses[b] if poses is not None else (np.zeros(2), 0.0)
            histories[b].push(fused, loc, ori)
        # (3) stack t, t-5, t-10 into the batch buffer
        sel = [h.selected() for h in histories]
        counts = [sum(s[0].shape[0] for s in ss) for ss in sel]
        P = max(counts)
        stacked = torch.empty((B, P, 8 + NUM_FRAME_STACK + 1), dtype=torch.float32, device=self.device)
        for b in range(B):
            stack_into(stacked[b], sel[b])
        # (4)-(6) LiDAR model, detections, motion forecast + plan
        out = im.forward_batch(stacked, counts, nxps, cmds)
        # (7) brake predictor on the stitched wide view + tele view (lav_agent_fast.py:257-262,318-321)
        if self.bra_model is not None and tel_u8 is not None:
            out["pred_bra"] = brake_probs(self.bra_model, rgbs_u8, tel_u8, u8=False)
        return out


class StaticFramePipeline(FramePipeline):
    """Fixed-shape variant for throughput: B agents, N points per sweep (shorter sweeps are padded with NaN rows, which
    every kernel drops), all buffers static, the whole tick captured in two CUDA graphs:
      G1: seg -> batched paint -> table-driven stack -> pillars -> backbone -> heads -> peak extraction -> brake
      G2[Kb]: crops -> embed -> GRU roll-outs for the K detected vehicles + B egos.  K varies tick by tick (0 .. 15 B in real
             driving), so K is padded to the next multiple of K_BUCKET with dummy crops whose outputs are dropped: at most
             15 B / K_BUCKET + 1 distinct graphs exist, they share ONE memory pool, and an LRU keeps G2_CACHE of them.
    Between them the detections are decoded on the host exactly like InferModel.det_inference (one small D2H).
    The sweep FIFO of lav_agent_fast.py:267-274 is a device ring buffer; which slots feed the stack kernel is data in
    a device job table, so the captured graph never changes."""

    KEEP = NUM_FRAME_STACK * GAP + 1          # ticks t .. t-10
    K_BUCKET = 8                              # detected-vehicle counts are padded to a multiple of this
    G2_CACHE = 6                              # captured G2 graphs kept (least recently used is dropped)
    COPY_STREAM = os.environ.get("LAVB_COPY_STREAM", "1") != "0"   # stage pinned host inputs on a copy stream (see begin())

    def __init__(self, seg_model, lidar_model, uniplanner, bra_model, batch, n_points, camera_x=1.5, camera_z=2.4,
                 device=torch.device("cuda"), precision="f16", use_graphs=True, roof_filter=False, navigator=None):
        """roof_filter: the sweeps handed to step() are RAW sensor sweeps; the ego-roof drop of LAVAgent.preprocess
        (lav_agent_fast.py:247) then runs on the device as the first kernel of G1 (order preserving, NaN-padded).
        navigator: an AgentNavigator of the same B agents; begin(..., gnss=, compass=) then runs its front before G1 and feeds its
        commands and targets to the planner and its poses to the sweep stack, all on the device."""
        super().__init__(seg_model, lidar_model, uniplanner, bra_model, camera_x, camera_z, device, precision)
        B, N, T = batch, n_points, NUM_FRAME_STACK + 1
        self.B, self.N, self.T, self.use_graphs = B, N, T, use_graphs
        self.roof_filter = roof_filter
        dev = device
        self.rgbs = torch.zeros((B, 3, 288, 256, 3), dtype=torch.uint8, device=dev)
        self.tels = torch.zeros((B, 192, 480, 3), dtype=torch.uint8, device=dev)
        self.lidar = torch.full((B, N, 4), float("nan"), device=dev)
        self.lidar_raw = torch.full((B, N, 4), float("nan"), device=dev) if roof_filter else self.lidar
        self.cur = torch.full((B, N, 8), float("nan"), device=dev)
        self.ring = torch.full((B, self.KEEP, N, 8), float("nan"), device=dev)
        self.ring_pose = np.zeros((B, self.KEEP, 3))                 # loc x, loc y, ori per slot
        self.ring_valid = np.zeros((B, self.KEEP), dtype=bool)
        if navigator is not None and navigator.B != B:
            raise ValueError(f"StaticFramePipeline: a navigator of {navigator.B} agents for {B}")
        self.navigator = navigator
        # with a navigator the poses the sweep stack reads live on the device (lavb_stack_job_poses); the host ring stays for the
        # host-pose path.  Host ticks copy their pose into the device ring; the first host tick after navigator ticks copies the
        # device ring back (one synchronising copy), so the two paths can alternate on one pipeline
        self.ring_pose_dev = torch.zeros((B, self.KEEP, 3), dtype=torch.float64, device=dev) if navigator is not None else None
        self._host_ring_stale = False
        self.stacked = torch.full((B, T * N, 8 + T), float("nan"), device=dev)
        self.jobs_host = torch.zeros(B * T * ops.STACK_JOB_DTYPE.itemsize, dtype=torch.uint8).pin_memory()
        self.jobs_dev = torch.zeros_like(self.jobs_host, device=dev)
        self.nxps = torch.zeros((B, 2), device=dev)
        self.cmds = torch.zeros((B,), dtype=torch.long, device=dev)
        self.tick = 0
        self.stream = torch.cuda.Stream(device=dev)
        # host inputs are staged by a copy stream into one of two buffer sets, so the H2D transfer of tick t+1 runs under the
        # planner graph of tick t instead of behind it on the compute stream (the graphs read fixed addresses: one D2D copy)
        self.copy_stream = torch.cuda.Stream(device=dev)
        self._stage = [None, None]
        self._stage_free = [None, None]
        self._g1 = None
        self._g2 = {}            # Kb -> (graph, outputs, static inputs); insertion order = recency (LRU)
        self._g2_pool = None     # one graph memory pool for every G2[Kb]
        self._launches = []      # lav_b200 kernel launches per captured graph (G1 first)
        self._cams = np.stack([c.packed() for c in self.infer_model.coord_converters])

    # ---- host-side state ------------------------------------------------------------------------------------
    def _fill_jobs(self, poses, device_poses=False):
        """rewrite the (agent, sweep) job table for this tick — vectorised numpy, then one small H2D copy.  With device_poses the
        pose fields (R, dx, dy) are left for lavb_stack_job_poses to write after the copy."""
        B, T, N, KEEP = self.B, self.T, self.N, self.KEEP
        jobs = self.jobs_host.numpy().view(ops.STACK_JOB_DTYPE).reshape(B, T)
        s0 = self.tick % KEEP
        if device_poses:
            pass
        elif poses is not None:
            self.ring_pose[:, s0, :2] = np.asarray([p[0] for p in poses], dtype=np.float64)
            self.ring_pose[:, s0, 2] = np.asarray([p[1] for p in poses], dtype=np.float64)
        else:
            self.ring_pose[:, s0] = 0
        self.ring_valid[:, s0] = True
        ticks = self.tick - np.arange(T) * GAP                                   # (T,)
        slots = ticks % KEEP
        valid = (ticks >= 0)[None] & self.ring_valid[:, slots]
        if not device_poses:
            pose = self.ring_pose[:, slots]                                       # (B,T,3)
            loc0, ori0 = pose[:, :1, :2], pose[:, :1, 2]
            d = pose[..., 2] - ori0                                               # (B,T)
            c0, si0 = np.cos(ori0), np.sin(ori0)
            dl = pose[..., :2] - loc0
            R = np.zeros((B, T, 9), dtype=np.float32)
            R[..., 0], R[..., 1], R[..., 3], R[..., 4], R[..., 8] = np.cos(d), np.sin(d), -np.sin(d), np.cos(d), 1.0
            jobs["R"] = R
            jobs["dx"] = dl[..., 0] * c0 + dl[..., 1] * si0                       # dloc @ [[c,-s],[s,c]]
            jobs["dy"] = -dl[..., 0] * si0 + dl[..., 1] * c0
        jobs["n"] = np.where(valid, N, 0)
        jobs["time_idx"] = np.arange(T)[None]
        row_bytes = 4 * (8 + T)
        ring_b, ring_s = self.ring.stride(0) * 4, self.ring.stride(1) * 4
        src = self.ring.data_ptr() + np.arange(B, dtype=np.uint64)[:, None] * np.uint64(ring_b) + slots.astype(np.uint64)[None] * np.uint64(ring_s)
        src[:, 0] = self.cur.data_ptr() + np.arange(B, dtype=np.uint64) * np.uint64(self.cur.stride(0) * 4)
        jobs["src"] = src
        jobs["dst"] = (self.stacked.data_ptr() + np.arange(B, dtype=np.uint64)[:, None] * np.uint64(self.stacked.stride(0) * 4)
                       + np.arange(T, dtype=np.uint64)[None] * np.uint64(N * row_bytes))
        self.jobs_dev.copy_(self.jobs_host, non_blocking=True)

    def preload_history(self, b, sweeps):
        """test/bench helper: sweeps = [(fused (n,8), loc, ori)] for ticks t-1, t-2, ... relative to the NEXT step."""
        for k, (s, loc, ori) in enumerate(sweeps, 1):
            t = self.tick - k
            slot = t % self.KEEP
            self.ring[b, slot].fill_(float("nan"))
            self.ring[b, slot, :s.shape[0]] = s
            self.ring_pose[b, slot] = (loc[0], loc[1], ori)
            if self.ring_pose_dev is not None:
                self.ring_pose_dev[b, slot] = torch.from_numpy(self.ring_pose[b, slot].copy())
            self.ring_valid[b, slot] = True

    # ---- device work ----------------------------------------------------------------------------------------
    def _g1_body(self):
        B, N = self.B, self.N
        im = self.infer_model
        # the brake predictor only needs the camera frames: fork it onto a side stream so its (cuDNN) kernels fill the
        # tails of the perception kernels; inside a captured graph this becomes a parallel branch
        bra, side = None, None
        if self.bra_model is not None and FORK_BRAKE:
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                bra = self._brake()
        if self.roof_filter:
            ops.roof_filter(self.lidar_raw, pad_nan=True, out=self.lidar)
        if FUSE_SEG_HEAD:
            feat, table, ncls = self.seg_model.forward_features_nhwc(self.rgbs.view(B * 3, 288, 256, 3))
            ops.paint_deconv_batched(self.lidar, feat, ncls, table, self._cams, 4, self.cur, (288, 256))
        else:
            logits = self.seg_model.forward_nhwc(self.rgbs.view(B * 3, 288, 256, 3))
            logits = logits.view(B, 3, *logits.shape[1:]).permute(0, 1, 4, 2, 3)
            ops.paint_batched(self.lidar, logits, self._cams, 2, 4, self.cur)
        ops.stack_jobs(self.jobs_dev, B * self.T, N, 8, self.T)
        feats, center, box, ori, seg = im.lidar_model.forward_nhwc(self.stacked, [self.T * N] * B)
        packed = ops.det_peaks(center, box, ori)        # sigmoid + 7x7 NMS + top-15 + map reads in two small kernels
        heat = None
        if side is not None:
            torch.cuda.current_stream().wait_stream(side)
        elif self.bra_model is not None:
            bra = self._brake()
        return dict(features=feats, pred_bev=seg.permute(0, 3, 1, 2), packed=packed, pred_bra=bra, heat=heat)

    def _brake(self):
        return brake_probs(self.bra_model, self.rgbs, self.tels)

    def _g2_body(self, K, locs, oris, fidx):
        return self.infer_model.uniplanner.infer_device(self._o1["features"].permute(0, 3, 1, 2), locs, oris, fidx, K, self.nxps, self.cmds)

    def _capture(self, fn, pool=None):
        for _ in range(2):
            out = fn()                                       # warm-up: cuDNN plans, workspaces, plan caches
        torch.cuda.synchronize()
        c0 = ops.launches()
        if not self.use_graphs:
            out = fn()
            self._launches.append(ops.launches() - c0)
            return None, out
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=pool):
            out = fn()
        self._launches.append(ops.launches() - c0)      # lav_b200 kernels recorded in this graph
        return g, out

    @torch.no_grad()
    def step(self, rgbs_u8, tel_u8, lidars, nxps=None, cmds=None, poses=None, fixed_dets=None, gnss=None, compass=None):
        """rgbs_u8 (B,3,288,256,3) u8 / tel_u8 (B,192,480,3) u8 on host (pinned) or device; lidars: (B,n,4) tensor or list of
        (n_b,4) (n_b <= N); nxps (B,2); cmds (B,) ints; or, with a navigator, gnss and compass instead (see begin).  Returns the
        dict of FramePipeline.step.
        = begin() + finish(); call them separately to overlap the host-side decode of one pipeline with the GPU work of
        another (each StaticFramePipeline owns a stream)."""
        self.begin(rgbs_u8, tel_u8, lidars, nxps, cmds, poses, gnss=gnss, compass=compass)
        return self.finish(fixed_dets)

    @torch.no_grad()
    def begin(self, rgbs_u8, tel_u8, lidars, nxps=None, cmds=None, poses=None, gnss=None, compass=None):
        """stage inputs and launch G1 (asynchronous).  With gnss ((B, >=2) lat, lon) and compass ((B,) raw imu[-1]) the navigator's
        front runs first, on the device: its cmds and nxps feed the planner, its poses the sweep stack, and nxps / cmds / poses
        must be None.  Returns the front's dict (AgentNavigator.front) then, else None."""
        nav = None
        if gnss is not None or compass is not None:
            if self.navigator is None or gnss is None or compass is None:
                raise ValueError("StaticFramePipeline.begin: gnss and compass need a navigator and each other")
            if nxps is not None or cmds is not None or poses is not None:
                raise ValueError("StaticFramePipeline.begin: nxps, cmds and poses come from the navigator when gnss is given")
        elif nxps is None or cmds is None:
            raise ValueError("StaticFramePipeline.begin: nxps and cmds, or gnss and compass, are needed")
        rgbs_u8, tel_u8, lidars, used = self._stage_host(rgbs_u8, tel_u8, lidars)
        with torch.cuda.stream(self.stream), self._math_mode():
            if gnss is not None:
                nav = self.navigator.front(gnss, compass, out=dict(nxps=self.nxps))
            self._begin(rgbs_u8, tel_u8, lidars, nxps, cmds, poses, nav)
            if used is not None:
                self._stage_free[used] = torch.cuda.Event()
                self._stage_free[used].record(self.stream)
        return nav

    def _stage_host(self, rgbs_u8, tel_u8, lidars):
        """pinned host tensors -> the staging set of this tick on the copy stream; returns device tensors (or the arguments
        unchanged when they are already on the device / ragged) and the staging slot used."""
        full = torch.is_tensor(lidars) and lidars.shape[1] == self.N
        host = [t for t in (rgbs_u8, tel_u8, lidars if full else None) if torch.is_tensor(t) and t.device.type == "cpu" and t.is_pinned()]
        if not host or not self.COPY_STREAM:
            return rgbs_u8, tel_u8, lidars, None
        k = self.tick % 2
        if self._stage[k] is None:
            self._stage[k] = (torch.empty_like(self.rgbs), torch.empty_like(self.tels), torch.empty_like(self.lidar_raw))
        out = [rgbs_u8, tel_u8, lidars]
        with torch.cuda.stream(self.copy_stream):
            if self._stage_free[k] is not None:
                self.copy_stream.wait_event(self._stage_free[k])          # the tick that last read this set has consumed it
            for j, t in enumerate(out):
                if any(t is h for h in host):
                    self._stage[k][j].copy_(t, non_blocking=True)
                    out[j] = self._stage[k][j]
            ready = torch.cuda.Event()
            ready.record(self.copy_stream)
        self.stream.wait_event(ready)
        return out[0], out[1], out[2], k

    @torch.no_grad()
    def finish(self, fixed_dets=None):
        """decode detections on the host, launch G2, return the outputs (device tensors, valid on self.stream)."""
        with torch.cuda.stream(self.stream), self._math_mode():
            out = self._finish(fixed_dets)
        torch.cuda.current_stream().wait_stream(self.stream)
        return out

    def _begin(self, rgbs_u8, tel_u8, lidars, nxps, cmds, poses, nav=None):
        B, N = self.B, self.N
        self.rgbs.copy_(rgbs_u8, non_blocking=True)
        if tel_u8 is not None:
            self.tels.copy_(tel_u8, non_blocking=True)
        if torch.is_tensor(lidars) and lidars.shape[1] == N:
            self.lidar_raw.copy_(lidars, non_blocking=True)
        else:
            for b, l in enumerate(lidars):
                self.lidar_raw[b, :l.shape[0]].copy_(l, non_blocking=True)
                if l.shape[0] < N:
                    self.lidar_raw[b, l.shape[0]:].fill_(float("nan"))
        if nav is None:
            self.nxps.copy_(torch.as_tensor(nxps, dtype=torch.float32), non_blocking=True)
            self.cmds.copy_(torch.as_tensor(cmds, dtype=torch.long), non_blocking=True)
            if self._host_ring_stale:
                self.ring_pose[:] = self.ring_pose_dev.cpu().numpy()
                self._host_ring_stale = False
            self._fill_jobs(poses)
            if self.ring_pose_dev is not None:       # keep the device ring whole for later navigator ticks
                s0 = self.tick % self.KEEP
                self.ring_pose_dev[:, s0].copy_(torch.from_numpy(self.ring_pose[:, s0].copy()), non_blocking=True)
        else:                                        # the front wrote self.nxps; its poses go to the ring and the job table
            self.cmds.copy_(nav["cmds"])
            self._fill_jobs(None, device_poses=True)
            ops.stack_job_poses(self.jobs_dev, self.B, self.T, GAP, self.KEEP, self.tick, self.ring_pose_dev, nav["poses"])
            self._host_ring_stale = True
        if self._g1 is None:
            self._g1, self._o1 = self._capture(self._g1_body)
        if self._g1 is not None:
            self._g1.replay()
        else:
            self._o1 = self._g1_body()
        self.ring[:, self.tick % self.KEEP].copy_(self.cur)                   # FIFO push (lav_agent_fast.py:267)
        self.tick += 1

    def _finish(self, fixed_dets):
        B = self.B
        o1 = self._o1
        dets = self.infer_model.decode_packed(o1["packed"])
        veh = [list(fixed_dets) for _ in range(B)] if fixed_dets is not None else [d[1] for d in dets]
        up = self.infer_model.uniplanner
        H, W = o1["features"].shape[1] * 2, o1["features"].shape[2] * 2
        locs, oris, fidx, counts = [], [], [], []
        for b in range(B):
            l, o = up.det_to_locs(veh[b], H, W)
            locs += l; oris += o; fidx += [b] * len(l); counts.append(len(l))
        K = len(locs)
        Kb = -(-K // self.K_BUCKET) * self.K_BUCKET          # rows K..Kb are dummy crops (frame 0, origin), outputs dropped
        if Kb in self._g2:
            self._g2[Kb] = self._g2.pop(Kb)                  # mark most recently used
        else:
            if len(self._g2) >= self.G2_CACHE:
                self._g2.pop(next(iter(self._g2)))           # evict the least recently used graph (its blocks return to the pool)
            if self._g2_pool is None and self.use_graphs:
                self._g2_pool = torch.cuda.graph_pool_handle()
            st = dict(locs=torch.zeros((Kb + B, 2), device=self.device), oris=torch.zeros((Kb + B,), device=self.device),
                      fidx=torch.zeros((Kb + B,), dtype=torch.int32, device=self.device))
            st["fidx"][Kb:] = torch.arange(B, dtype=torch.int32, device=self.device)
            g, out = self._capture(lambda: self._g2_body(Kb, st["locs"], st["oris"], st["fidx"]), pool=self._g2_pool)
            self._g2[Kb] = (g, out, st)
        g, out, st = self._g2[Kb]
        if K > 0:
            pk = torch.tensor([l + [o, float(f)] for l, o, f in zip(locs, oris, fidx)], dtype=torch.float32).to(self.device, non_blocking=True)
            st["locs"][:K].copy_(pk[:, :2]); st["oris"][:K].copy_(pk[:, 2]); st["fidx"][:K].copy_(pk[:, 3])
        if g is not None:
            g.replay()
        else:
            out = self._g2_body(Kb, st["locs"], st["oris"], st["fidx"])
        ee, epl, ecl, ocl, occ = out
        ocl, occ = ocl[:K], occ[:K]
        return dict(ego_embd=ee, ego_plan_locs=epl, ego_cast_locs=ecl, other_cast_locs=torch.split(ocl, counts),
                    other_cast_cmds=torch.split(occ, counts), pred_bev=o1["pred_bev"], det=dets, features=o1["features"],
                    pred_bra=o1["pred_bra"])

"""The agent's debug view on the GPU: the frame LAVAgent.run_step draws and keeps every tick (team_code_v2/lav_agent_fast.py:354-358,
visualize :459-518) for B agents, bit for bit with the reference's numpy and OpenCV drawing, and the recorder that collects the
frames per agent as flush_data (:160-167) does.

    view = AgentView(B, config)                      # config: the agent's loaded YAML dict
    rec = AgentRecorder(view)
    out = pipeline.finish()                          # StaticFramePipeline
    res = ctl.step(out, speeds, pipeline.cmds)       # AgentController
    rec.record(pipeline, out, res, speeds)           # no host synchronisation
    ...
    frames = rec.flush([i])[i]                       # (T, 160, 1146, 3) uint8 of agent i, annotated, then cleared

render() gives the frames without their text, as a (B, 160, 1146, 3) uint8 device tensor; annotate() writes visualize's four text
lines on host frames with cv2.putText.  Video encoding and upload stay with the caller.
"""
import queue
import threading

import numpy as np
import torch

from . import capi, ops

CONFIG_KEYS = ("pixels_per_meter", "cmd_thresh")
FRAME_SHAPE = (160, 1146, 3)
FLUSH_FRAMES = 12000                                 # run_step flushes an agent's frames at this many (lav_agent_fast.py:360)
CMD_NAMES = {0: 'left', 1: 'right', 2: 'straight', 3: 'follow', 4: 'change left', 5: 'change right'}

# matplotlib's _jet_data: (x, y0, y1) per segment of each channel
_JET = (((0., 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1, 0.5, 0.5)),
        ((0., 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.64, 1, 1), (0.91, 0, 0), (1, 0, 0)),
        ((0., 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1, 0, 0)))


def jet_bytes(n=256):
    """(n + 3, 3) uint8: visualize's (int(r * 255), int(g * 255), int(b * 255)) of matplotlib's jet (LinearSegmentedColormap
    of _jet_data with n colours, _create_lookup_table with gamma 1), then its under, over and bad rows (first colour, last
    colour, black)."""
    lut = np.zeros((n + 3, 3))
    for j, seg in enumerate(_JET):
        a = np.array(seg, dtype=np.float64)
        x, y0, y1 = a[:, 0] * (n - 1), a[:, 1], a[:, 2]
        xind = (n - 1) * np.linspace(0, 1, n) ** 1.0
        ind = np.searchsorted(x, xind)[1:-1]
        distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
        lut[:n, j] = np.clip(np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0.0, 1.0)
    lut[n], lut[n + 1], lut[n + 2] = lut[0], lut[n - 1], 0.0
    return (lut * 255).astype(np.int64).astype(np.uint8)


def view_config(config):
    """the capi.ViewConfig of the agent's YAML dict; a missing key is an error."""
    missing = [k for k in CONFIG_KEYS if k not in config]
    if missing:
        raise KeyError(f"agent config lacks {missing}")
    c = capi.ViewConfig()
    c.pixels_per_meter, c.cmd_thresh = float(config["pixels_per_meter"]), float(config["cmd_thresh"])
    c.jet[:] = jet_bytes().reshape(-1).tolist()
    return c


def box_table(dets):
    """the vehicle boxes det[1] of each agent's detections (InferModel.decode_packed's lists) as the (NB, 6) fp64 table and the
    (B + 1,) int32 offsets agent_view takes."""
    rows = [list(d[1]) for d in dets]
    offsets = np.zeros(len(rows) + 1, dtype=np.int32)
    np.cumsum([len(r) for r in rows], out=offsets[1:])
    table = np.array([box for r in rows for box in r], dtype=np.float64).reshape(-1, 6)
    return table, offsets


def annotate(frames, speeds, cmds, control, pred_bra):
    """visualize's four cv2.putText lines on host frames (B, 160, 1146, 3) uint8, in place: speed (m/s), the command, steer /
    throttle / brake and the brake model's probability of each agent."""
    import cv2
    args = (cv2.FONT_HERSHEY_SIMPLEX, 0.3, (255, 255, 255), 1)
    speeds, cmds = np.asarray(speeds).reshape(-1), np.asarray(cmds).reshape(-1)
    control, pred_bra = np.asarray(control).reshape(-1, 3), np.asarray(pred_bra).reshape(-1)
    for i, f in enumerate(frames):
        steer, throt, brake = control[i]
        cv2.putText(f, f'speed: {speeds[i]:.3f}m/s', (4, 10), *args)
        cv2.putText(f, 'cmd: {}'.format(CMD_NAMES.get(int(cmds[i]))), (4, 30), *args)
        cv2.putText(f, f'steer: {steer:.3f} throttle: {throt:.3f} brake: {brake:.3f}', (4, 20), *args)
        cv2.putText(f, f'predicted brake: {pred_bra[i]:.3f}', (4, 40), *args)
    return frames


class AgentView:
    """Debug frames of ``batch`` agents on ``device``."""

    def __init__(self, batch, config, device=torch.device("cuda")):
        self.B = int(batch)
        self.config = view_config(config)
        self.device = torch.device(device)
        self.scratch = torch.empty((ops.agent_view_scratch_bytes(self.B),), dtype=torch.uint8, device=self.device)

    def render(self, pipeline, out):
        """One tick's frames, (B, 160, 1146, 3) uint8 on the current stream.  pipeline: the StaticFramePipeline of these agents,
        whose cameras, stacked sweeps, commands and targets of the tick are read; out: its finish() dict (plans, forecasts,
        pred_bev, det).  The pipeline's stream waits for the frames, so its next tick cannot overwrite what they read."""
        B = self.B
        if pipeline.B != B:
            raise capi.LavbError(f"AgentView.render: a pipeline of {pipeline.B} agents for {B}")
        ocl, occ = list(out["other_cast_locs"]), list(out["other_cast_cmds"])
        if len(ocl) != B or len(occ) != B or len(out["det"]) != B:
            raise capi.LavbError(f"AgentView.render: {len(ocl)} forecast groups and {len(out['det'])} detections for {B} agents")
        offsets = np.zeros(B + 1, dtype=np.int32)
        np.cumsum([len(o) for o in ocl], out=offsets[1:])
        boxes, box_offsets = box_table(out["det"])
        f32 = lambda t: t.to(torch.float32).contiguous()
        frames = ops.agent_view(pipeline.rgbs, pipeline.tels, pipeline.stacked, out["pred_bev"], f32(out["ego_plan_locs"]),
                                f32(out["ego_cast_locs"]), pipeline.cmds.to(torch.int32), f32(torch.cat(ocl)), f32(torch.cat(occ)),
                                offsets, boxes, box_offsets, pipeline.nxps, self.config, self.scratch)
        pipeline.stream.wait_stream(torch.cuda.current_stream())
        return frames


class AgentRecorder:
    """Collects each agent's annotated frames as run_step and flush_data do.  record() renders the tick and copies the frames
    and the text values into pinned memory on a side stream behind an event, so the tick is not synchronised; a writer thread
    waits for the copy, annotates the frames and appends them per agent.  flush(agents) hands out and clears their frames."""

    def __init__(self, view, depth=4):
        self.view = view
        self.B = view.B
        self.frames = [[] for _ in range(self.B)]
        self.copy_stream = torch.cuda.Stream(device=view.device)
        self._free = queue.Queue()
        for _ in range(depth):                          # pinned slots: frames and text values of one tick each
            self._free.put(dict(frames=torch.empty((self.B, *FRAME_SHAPE), dtype=torch.uint8).pin_memory(),
                                text=torch.empty((self.B, 5), dtype=torch.float32).pin_memory(),
                                cmds=torch.empty((self.B,), dtype=torch.int32).pin_memory()))
        self._work = queue.Queue()
        self._lock = threading.Lock()
        self._error = None
        self._thread = threading.Thread(target=self._write, daemon=True)
        self._thread.start()

    def record(self, pipeline, out, res, speeds):
        """render this tick's frames and queue them: res is AgentController.step's result (its controls), speeds (B,) m/s as a
        host array or a device tensor.  Returns the device frames (valid on the current stream)."""
        self._raise()
        dev = self.view.device
        frames = self.view.render(pipeline, out)
        speed = speeds.to(dev, torch.float32) if torch.is_tensor(speeds) else torch.as_tensor(np.asarray(speeds, np.float32), device=dev)
        text = torch.cat([speed.reshape(self.B, 1), res["control"].reshape(self.B, 3).float(),
                          out["pred_bra"].reshape(self.B, 1).float()], 1)
        cmds = pipeline.cmds.to(torch.int32)
        slot = self._free.get()
        self.copy_stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.copy_stream):
            slot["frames"].copy_(frames, non_blocking=True)
            slot["text"].copy_(text, non_blocking=True)
            slot["cmds"].copy_(cmds, non_blocking=True)
            done = torch.cuda.Event()
            done.record(self.copy_stream)
        for t in (frames, text, cmds):                  # keep the device sources alive until the copy has read them
            t.record_stream(self.copy_stream)
        self._work.put((slot, done))
        return frames

    def _write(self):
        while True:
            item = self._work.get()
            if item is None:
                return
            slot, done = item
            try:
                done.synchronize()
                f = slot["frames"].numpy().copy()
                x, c = slot["text"].numpy(), slot["cmds"].numpy()
                annotate(f, x[:, 0], c, x[:, 1:4], x[:, 4])
                with self._lock:
                    for i in range(self.B):
                        self.frames[i].append(f[i])
            except Exception as e:        # surfaced by the next record / flush
                self._error = e
            finally:
                self._free.put(slot)
                self._work.task_done()

    def _raise(self):
        if self._error is not None:
            e, self._error = self._error, None
            raise e

    def pending(self, agent):
        """frames of ``agent`` collected so far (after the queued ticks are written)."""
        self._work.join()
        with self._lock:
            return len(self.frames[agent])

    def flush(self, agents=None):
        """{agent: (T, 160, 1146, 3) uint8} of ``agents`` (all when None), each agent's frames cleared, as flush_data does at
        route end or every FLUSH_FRAMES frames; waits for the queued ticks first."""
        self._work.join()
        self._raise()
        agents = range(self.B) if agents is None else agents
        out = {}
        with self._lock:
            for i in agents:
                out[i] = np.stack(self.frames[i]) if self.frames[i] else np.zeros((0, *FRAME_SHAPE), np.uint8)
                self.frames[i] = []
        return out

    def close(self):
        """stop the writer thread (queued ticks are written first)."""
        self._work.put(None)
        self._thread.join()

"""The agent's controls on the GPU: the decision tail of LAVAgent.run_step (team_code_v2/lav_agent_fast.py:228-231, 325-352) for
B agents — the stop counter, the 4/5 plan swap, the two PID controllers of pid_control (called twice per tick, :404-426,
team_code_v2/pid.py), plan_collide's safety brake (:385-401), the brake model's threshold, the speed cap and the creep after a
long stop — in one lavb_agent_control launch per tick, with every agent's controller state resident on the device.

    ctl = AgentController(B, config)                 # config: the agent's loaded YAML dict
    out = pipeline.step(...)                         # FramePipeline.step / StaticFramePipeline.finish
    res = ctl.step(out, speeds, cmds)                # on the current stream, no host synchronisation
    steer, throttle, brake = res["control"].cpu()[i]    # the one copy the EKF and carla.VehicleControl need

Flags per agent (res["flags"], int32) are the FLAG_* bits below.
"""
import numpy as np
import torch

from . import capi, ops

# the keys of the agent's YAML config the controls read (team_code_v2/config.yaml: the CONTROLLER section, cmd_thresh,
# pixels_per_meter)
CONFIG_KEYS = ("aim_point", "speed_ratio", "turn_KP", "turn_KI", "turn_KD", "turn_n", "speed_KP", "speed_KI", "speed_KD",
               "speed_n", "brake_speed", "clip_delta", "max_throttle", "max_speed", "cmd_thresh", "pixels_per_meter")
# LAVB_CTL_* of include/lav_b200.h
FLAG_PLAN_INVALID, FLAG_PID_BRAKE, FLAG_BRAKE_MODEL, FLAG_COLLIDE, FLAG_SPEED_CAP, FLAG_CREEP, FLAG_BAD_CMD = 1, 2, 4, 8, 16, 32, 64
MAX_CMDS = 8


def control_config(config):
    """the capi.ControlConfig of the agent's YAML dict; a missing key is an error."""
    missing = [k for k in CONFIG_KEYS if k not in config]
    if missing:
        raise KeyError(f"agent config lacks {missing}")
    c = capi.ControlConfig()
    aim, ratio = list(config["aim_point"]), list(config["speed_ratio"])
    if not 1 <= len(aim) <= MAX_CMDS or len(ratio) != len(aim):
        raise capi.LavbError(f"agent config: aim_point ({len(aim)}) and speed_ratio ({len(ratio)}) need one entry per command, "
                             f"at most {MAX_CMDS}")
    for j, (a, r) in enumerate(zip(aim, ratio)):
        c.aim_point[j], c.speed_ratio[j] = int(a), float(r)
    c.turn_kp, c.turn_ki, c.turn_kd = float(config["turn_KP"]), float(config["turn_KI"]), float(config["turn_KD"])
    c.speed_kp, c.speed_ki, c.speed_kd = float(config["speed_KP"]), float(config["speed_KI"]), float(config["speed_KD"])
    c.turn_n, c.speed_n = int(config["turn_n"]), int(config["speed_n"])
    for k in ("brake_speed", "clip_delta", "max_throttle", "max_speed", "cmd_thresh", "pixels_per_meter"):
        setattr(c, k, float(config[k]))
    return c


class AgentController:
    """Controller state and per-tick controls of ``batch`` agents on ``device``."""

    def __init__(self, batch, config, device=torch.device("cuda")):
        self.B = int(batch)
        self.config = control_config(config)
        self.num_cmds = len(config["aim_point"])
        self.device = torch.device(device)
        self.record = ops.agent_control_state_bytes(self.config.turn_n, self.config.speed_n)
        self.state = torch.zeros((self.B * self.record,), dtype=torch.uint8, device=self.device)

    def reset(self, agents=None):
        """a new route for ``agents`` (all when None): their PID windows and counters back to zero; no other agent changes."""
        rows = self.state.view(self.B, self.record)
        if agents is None:
            rows.zero_()
        else:
            idx = torch.as_tensor(np.asarray(agents, dtype=np.int64).reshape(-1))
            if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= self.B):
                raise IndexError(f"reset: agents {idx.tolist()} outside 0..{self.B - 1}")
            rows[idx.to(self.device)] = 0

    def step(self, out, speeds, cmds):
        """One tick.  out: the dict FramePipeline.step / StaticFramePipeline.finish returns (ego_plan_locs, ego_cast_locs,
        other_cast_locs, other_cast_cmds, pred_bra; read, never changed); speeds (B,) m/s, host values or a device tensor; cmds
        (B,) the commands the planner was given, host ints or an int32 device tensor (AgentNavigator.front's "cmds"; an agent
        whose command is outside the planner's branches gets NaN controls and FLAG_BAD_CMD).  -> dict(control (B,3) fp32 = steer, throttle, brake; flags (B,)
        int32), device tensors on the current stream."""
        B, dev = self.B, self.device
        ocl, occ = list(out["other_cast_locs"]), list(out["other_cast_cmds"])
        if len(ocl) != B or len(occ) != B:
            raise capi.LavbError(f"AgentController.step: {len(ocl)} forecast groups for {B} agents")
        offsets = np.zeros(B + 1, dtype=np.int32)
        np.cumsum([len(o) for o in ocl], out=offsets[1:])
        locs, scores = torch.cat(ocl), torch.cat(occ)                  # the rows of all agents, concatenated on the device
        if locs.shape[1] != self.num_cmds:
            raise capi.LavbError(f"AgentController.step: {locs.shape[1]} forecast branches for {self.num_cmds} commands")
        if torch.is_tensor(cmds) and cmds.is_cuda:                      # AgentNavigator.front's commands, read on the device
            cmds = cmds.to(torch.int32).reshape(-1).contiguous()
        else:
            cmds = np.asarray(cmds.numpy() if torch.is_tensor(cmds) else cmds).astype(np.int32).reshape(-1)
        if torch.is_tensor(speeds) and speeds.is_cuda:
            speed = speeds.to(torch.float32).reshape(B).contiguous()
        else:
            host = torch.as_tensor(np.asarray(speeds, dtype=np.float32).reshape(B))
            speed = host.pin_memory().to(dev, non_blocking=True)
        pred_bra = out["pred_bra"].reshape(B).to(torch.float32).contiguous()
        control, flags = ops.agent_control(out["ego_plan_locs"].contiguous(), out["ego_cast_locs"].contiguous(), locs.contiguous(),
                                           scores.contiguous(), offsets, pred_bra, speed, cmds, self.config, self.state)
        return dict(control=control, flags=flags)

    def state_views(self):
        """a host copy of the controller state (synchronises): stop / creep counters and the PID windows, oldest value first
        (ops.agent_control_state_views)."""
        return ops.agent_control_state_views(self.state.cpu().numpy(), self.config.turn_n, self.config.speed_n)

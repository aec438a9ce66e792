"""Score LiDAR and planner checkpoints on a held-out recording: the comparisons LAV.train_lidar draws for wandb
(lav/lav_final_v2.py:226-258) — predicted BEV against the recorded one, detections against the recorded actors, the ego plan
against the expert's future — as numbers over every sample of the recording, through the agent's eval-mode inference path.

    python -m lav_b200.evaluate --config-path config_v2.yaml --data-dir VALDIR --lidar-weights lidar_7.th \
        --uniplanner-weights uniplanner_7.th [--batch-size 32] [--precision f16|fp32] [--num-workers 16] [--json out.json] \
        [--forecast] [--forecast-detected] [--plan-safety] [--det-boxes] [--brake --bra-weights bra.th [--agent-config AGENT.yaml]] \
        [--seg-weights seg_1.th] [--driving-score [--step-seconds 0.25]]
    python -m lav_b200.evaluate ... --lidar-weights lidar_8.th lidar_16.th --uniplanner-weights uniplanner_8.th uniplanner_16.th
    python -m lav_b200.evaluate ... --run-dir RUN [--epochs 1,8,16-64]
    torchrun --nproc-per-node N -m lav_b200.evaluate ...

Every sample is taken once, in index order, unaugmented (TemporalBatchLoader's ordered mode); the last batch may be short.  Per
batch, InferModel.forward_batch runs the models and one ops.eval_batch launch scores its outputs; the one device-to-host copy
is that launch's result buffer.  The host sums the counts and computes AP over the whole recording.

Several checkpoints (weight paths paired by position, or train_full's lidar_{e}.th / uniplanner_{e}.th pairs found by --run-dir)
are scored in one pass, each batch loaded once and run through every checkpoint (evaluate_checkpoints, lav_b200.eval_sweep);
each checkpoint's result is exactly what a run of it alone reports.  One checkpoint prints and writes what a single run always
has; a sweep prints one row of headline numbers per checkpoint and writes {samples, ranks, checkpoints: [{epoch, weights,
result}]}.  Under torchrun each rank scores a contiguous range of the recording on GPU LOCAL_RANK % device_count and rank 0
merges the per-sample records over gloo, so the result is the one a single process computes from the same per-sample values;
rank 0 alone prints and writes --json.  The model outputs themselves are not bit-reproducible across runs (the pillar encoder
sums with float atomics), and a rank's LiDAR shuffle stream starts at its own first sample, so a sample's point order differs
from a single process's, and which points are kept differs when its sweep stack exceeds max_lidar_points.

Metrics:
  bev_iou[c]      intersection / union of (pred > 0.5, gt != 0) over all pixels of BEV channel c (null without any union)
  det[cls].ap[t]  all-point-interpolated AP of class cls (pedestrian, vehicle) at centre distance t metres: the surviving
                  detections of the recording sorted by descending score (ties keep sample order, then column order), the
                  precision envelope summed over the recall steps; null for a class with no actor in the window; "mean" is the
                  mean over the thresholds
  plan            ADE (mean over the steps of the Euclidean error) and FDE (error at the last step) in metres, over all samples
                  and per recorded command

With --forecast (``forecast=True``) the result also holds ``forecast``: the UniPlanner's motion forecasts scored by
ops.forecast_eval, one launch and one result copy per batch, from the LiDAR features forward_batch already computed.  The
protocol, shared with lav_b200.evaluate_bev (the privileged BEV planner):

  The forecasts are made from the recorded poses, which is what the training forward of both planners does with the jitter set
  to zero.
  Rows.  A row is an actor of a sample that the training selection rule accepts, heads.vehicles_ahead(ego_locs, locs[:, 1:],
    typs[:, 1:] == 1), in slot order.  The max_num_cars cap and its multinomial draw are not applied: every such actor is
    scored.  actor_tracks keeps only actors seen in all T + 1 frames, so every row has a full recorded future; padded slots have
    typ 0 and are never rows.
  Pose and target.  For a row at sample f and slot s >= 1 (slot 0 is the ego): start = locs[f, s, 0] - ego_locs[f, 0],
    heading = oris[f, s] - oris[f, 0], target = transform_points(locs[f, s, 1:] - locs[f, s, :1], -heading), in the actor's
    crop frame, the frame the loss compares in.  Ego rows use pose (0, 0) and target ego_locs[:, 1:].
  Models, in eval mode.  UniPlanner: crop of the LiDAR features at (start, heading), lidar_conv_emb at the agent's precision
    (the private copy agent.infer_model makes), then cast and cast_cmd_pred: infer_device's chain without its transform to the
    ego frame.  BEVPlanner: crop_u8_kernel crop of the uint8 ground-truth BEV at pixels_per_meter and 2 * crop_size, then
    bev_conv_emb, cast and cast_cmd_pred, in fp32 under math_mode("fp32"); its ego plan is
    plan(ego_embd, nxp, cast_locs=ego_cast)[:, -1].
  Metrics per row, with C branches and T steps; distances are fp64 Euclidean with no contraction.  ADE_j is the mean over t of
    |cast[j, t] - target[t]|, summed in ascending t and then divided by T; FDE_j is the error at t = T - 1.  minADE and minFDE
    are each minimised over j independently, ties to the lower j.  top is the branch with the highest command score, ties to
    the lower j, NaN counting as lowest; the row reports its ADE / FDE.  A row with a recorded command (ego rows) reports the
    ADE / FDE of that branch; rows without one (other vehicles, cmd = -1) get NaN there.
  Host reduction over the recording.  other: row count, mean minADE, mean minFDE, mean top-1 ADE and FDE, and miss rate
    (minFDE > 2 m).  ego_cast: ADE / FDE under the recorded command, minADE / minFDE, command accuracy (top == cmd), and the
    same per recorded command.  ego_plan (BEV planner only): the plan's ADE / FDE under the recorded command, overall and per
    command; the UniPlanner's plan is scored by ``plan`` above.  A mean over no row is null.

With --forecast-detected (``forecast_detected=True``) the result also holds ``forecast_detected``: the forecasts the agent acts
on, the ones UniPlanner.infer_batch makes for the vehicles the LiDAR model detects (other_cast_locs / other_cast_cmds of
forward_batch, the rows lav_agent_fast.plan_collide brakes on), matched to the recorded tracks and scored.  Per batch: one
ops.det_forecast_match launch and one ops.forecast_eval launch into the same buffer, that buffer copied to the host once, plus
one copy of the packed peaks (B x 7 x 30 floats) that the row table is built from; no extra model call.  The protocol:

  Rows.  A row is a detection infer_batch forecasts: a class-1 packed peak that passes decode_packed's filters
    (model_inference.peak_filter: score > float32(0.2) in fp32, the size filter, 2 px < d < 30 m) and det_to_locs' centre test
    (heads.off_centre: more than 4 px from the crop centre), in frame order, then packed-column order: the order of the
    concatenated other_cast_locs, whose per-frame lengths must equal the row counts.  The row table (frame, column) is built on
    the host (detected_rows) from a copy of the packed peaks.
  Ground truth.  eval_batch's vehicle class and window: the actor rows of the sample with typ == 1 whose centre (det_grid.cuh's
    det_centre) lies 2 px < d < 30 m from the ego.  Actor row a of a sample is label slot a (actor_tracks emits both in one id
    order, the labels capped at max_objs), so an actor has a recorded track when a < num_objs.
  Match.  Greedy per sample, the rows in eval_batch's order (descending score, then lower flat index, then lower column): each
    takes the nearest GT vehicle not yet taken whose centre is within match_m = 2 m (fp64 pixel distance, no contraction; equal
    distances to the lower actor row), the search eval_batch runs.  Vehicles without a track take part, so a detection of a
    capped actor never takes a tracked neighbour; rows matched to them are counted and not scored.
  Target.  For a row matched to a tracked actor a of sample f: locs[f, a, 1:] - ego_locs[f, 0] (the label tensors), the ego frame
    of other_cast_locs: det_to_locs maps a peak at (X, Y) to ((X - 160) / ppm, (Y - 280) / ppm), det_centre places an actor at
    X = -x * ppm + 160, and the labels are the negated actor positions.
  Metrics per row: ops.forecast_eval(other_cast_locs, other_cast_cmds, target, cmd = -1) as above (minADE, minFDE, the
    top-scored branch's ADE and FDE).
  Host reduction (DetectedForecastScores): rows; matched (to a tracked actor); matched_untracked; gt (tracked vehicles in the
    window); recall = matched / gt; over the matched rows the mean minADE, minFDE, top-1 ADE and FDE and the miss rate (minFDE >
    2 m); ap = average_precision over every row but the matched-untracked ones, ranked by detection score (ties keep sample, then
    column order), a row a true positive when matched to a tracked actor with minFDE <= 2 m, against gt; match_m.  A mean over
    no row, and recall and ap with gt = 0, are null.

Not scored: pedestrians (the planners forecast vehicles only).

With --plan-safety (``plan_safety=True``, also lav_b200.evaluate_bev) the result also holds ``plan_safety``: the open-loop
collision rate of the ego plan against the recorded (non-reactive) traffic and the share of plans that leave the road, the check
lav_agent_fast.plan_collide makes before the agent drives a plan.  Per batch: one ops.plan_safety launch and one copy of its
(B, 2, 8) int32 result; the actor table comes from the loader (datasets.plan_safety_table, built only when asked), the road from
the batch's bev; no extra model call.  The protocol:

  Trajectories.  n = 2 per sample, T steps in the label frame (that of ego_locs and ego_plan_locs, entry 0 of ego_locs the
    origin): the plan under the recorded command (evaluate: forward_batch's ego_plan_locs; evaluate_bev: the recorded command's
    branch of forecast_recorded's ego_plan, NaN when the command has no branch) and the expert, ego_locs[:, 1:].  The expert is
    scored by the same rules: it is the metric's floor on the recording and is always reported next to the plan.
  Ego box at step t = 1..T.  Centre p_t = traj[t - 1], p_0 the origin.  Heading d / sqrt(d . d), d = p_t - p_{t-1}, in fp64 with
    correctly rounded sqrt and divide (no trig); a step of less than 0.1 m keeps the previous heading, and the heading before
    step 1 is the ego's forward direction (0, -1) ("ahead" is negative y, heads.vehicles_ahead).  Half extents: the ego's
    recorded bbox at the sample's frame, read as CARLA's bounding_box.extent (half length along the heading, half width), the
    reading detections_to_heatmap's scaling of bbox by ppm implies; the synthetic ego's (2.4, 1.1) is a 4.8 x 2.2 m car.
  Actors.  Every actor of the sample's frame but the ego, with no radius filter and no max_objs cap.  It is present at step t
    when its id appears in frame index + t, with that frame's loc, ori, bbox and type; type 1 is a vehicle, 0 a pedestrian,
    others are ignored.  Positions go into the label frame as actor_tracks transforms them, then negated as the labels are.  A
    yaw psi relative to the ego heads along (sin psi, -cos psi) there: actor_tracks maps a world direction (cos phi, sin phi)
    through R = [[sin e, cos e], [-cos e, sin e]] (e the ego yaw) to (-sin psi, cos psi) with psi = phi - e, negated to
    (sin psi, -cos psi); psi = 0 gives the ego's own (0, -1).  cos psi and sin psi are computed on the host in fp64 and travel in the table.
  Collision.  A separating-axis test of the two rectangles over both boxes' headings and their perpendiculars (u2 = (-u1y,
    u1x)): on axis n the separation |(c_B - c_A) . n| against the reach r_A(n) + r_B(n), r(n) = e1 |u1 . n| + e2 |u2 . n|, in
    fp64 with no contraction, evaluated in the order written; separated when separation >= reach, so touching does not collide.
    A step collides with a class when any present actor of that class overlaps the ego box.
  Leaving the road.  The four corners of the ego box go to map pixels as det_centre places label-frame coordinates: column =
    floor(x * ppm + cx0), row = floor((y * ppm + cy0) + cy1), in fp64, i.e. (160 + 4x, 280 + 4y) on the v2 grid.  A corner
    outside the 320 x 320 map is off the map; a step is off-road when any in-map corner lands on a 0 pixel of bev[:, 0] (the road
    plane; in the ordered, unaugmented loaders it is in the label frame).  A step with a corner off the map counts in
    off_map_steps; its in-map corners still decide whether it is off-road.
  Invalid steps.  A step whose centre or heading is not finite (a NaN point also spoils the next step's heading) is counted in
    invalid_steps and is never a collision or off-road.
  Per sample and trajectory (ops.plan_safety_views): the first vehicle-collision step and the actor row it hit, the same for
    pedestrians, the first off-road step, off_map_steps and invalid_steps; steps are numbered 1..T, -1 for none.
  Host reduction (PlanSafetyScores), for plan and for expert, overall and per recorded command: samples, collision_rate (either
    class), vehicle_collision_rate, pedestrian_collision_rate, off_road_rate, collision_rate_by_step (T values: the share of
    samples whose first collision is at or before that step), and the summed off_map_steps and invalid_steps.  A rate over no
    sample is null.

With --driving-score (``driving_score=True``, also lav_b200.evaluate_bev) the result also holds ``driving_score``: a PDM-style
score of the same two trajectories, the open-loop stand-in for closed-loop driving that nuPlan and NAVSIM use, built from no
at-fault collision (NC), drivable-area compliance (DAC), time to collision (TTC), ego progress (EP) and comfort (C), against the
recorded, non-reactive traffic.  It ranks plans that plan ADE / FDE cannot: a plan that stops for a car that then runs into it
from behind keeps NC, and a plan that never moves loses EP.  Per batch: one ops.driving_score launch and one copy of its result
buffer; the actor table comes from the loader (datasets.driving_score_table, built only when asked), the road from the batch's
bev; no extra model call.  It works with or without --plan-safety.  The protocol:

  Trajectories, ego boxes, validity, actors, the collision test and the road rule are the plan-safety protocol's, unchanged
    (the plan under the recorded command and the expert ego_locs[:, 1:]; step 0 is the origin with heading (0, -1), headings
    carried over steps shorter than 0.1 m).  The actor table has one more step: step 0, the actors at the sample's own frame.
  Step period.  dt = --step-seconds (``step_seconds``), default 0.25 s.  The recordings carry no timestamps, so the default is
    inferred from the reference agent, not measured on a recording: the agent stacks sweeps GAP = NUM_REPEAT + 1 = 5 sensor
    ticks apart (team_code_v2/lav_agent_fast.py:32-33,150,368), its sensor tick is 0.05 s (:44), and training stacks
    consecutive recorded frames, so one recorded frame stands for 5 x 0.05 s.
  Velocities, t = 1..T, fp64.  Ego v_t = (p_t - p_{t-1}) / dt; the ego is stopped at t when |v_t| < 0.05 m/s.  An actor's
    velocity at t is (q_t - q_{t-1}) / dt from its step t - 1 and step t positions when it is present at both, else 0.
  NC.  A collision with actor a is new at step t when the boxes overlap at t and did not at t - 1 (at t = 1 the origin box
    against the actor's step-0 box; an actor absent at t - 1 did not overlap).  A new collision is not at fault when the ego is
    stopped or it is a rear collision, (q_t - p_t) . h_t < -e1 (the actor's centre behind the ego's rear face); every other
    new collision is at fault: front, lateral, or against a stopped actor.  nuPlan also exempts lateral collisions by the lanes
    the two agents occupy; the recordings have no lanes, so every lateral collision here is at fault.  NC = 0 if any at-fault
    collision with a vehicle or a pedestrian occurs, else 1.  An overlap already present at step 0 is never new.
  DAC.  0 if any valid step is off-road under the plan-safety corner rule, else 1: per sample the plan-safety off-road verdict.
  TTC.  At each step t where the ego is not stopped, every present actor that does not overlap the ego at t: both boxes are
    moved at constant velocity, headings held, to t + k dt, k = 1..K, K = floor(1.0 s / dt + 1e-9) (4 at 0.25 s); the ego to
    p_t + (k dt) v_t, the actor to q_t + (k dt) u_t.  The projected collision is judged at the first k whose boxes overlap,
    where it would begin: the step violates TTC unless the projected actor's centre is behind the projected ego's rear face
    there (the at-fault rule's rear exemption; the ego is moving).  TTC = 0
    if any step violates it, else 1.
  EP.  L = the arc length of the expert polyline, origin -> expert points, segment lengths summed in order; s = the arc-length
    position of the plan's last point projected onto that polyline: on each segment the closest point (the projection
    parameter clamped to [0, 1], 0 on a zero-length segment), the first segment of least distance, s = the segments before it +
    the parameter x its length.  EP = clamp(s / L, 0, 1), 0 when s / L is not a number; EP = 1 when L < 5 m (NAVSIM's
    minimum-progress rule).
  C.  Finite differences at dt, with no smoothing: nuPlan first smooths the trajectory with a Savitzky-Golay filter, this score
    does not, so a jagged plan fails more often than it would there; each term's failure rate is reported for that reason.
    Speed |v_t| (t >= 1); yaw psi_t = atan2 of h_t; yaw differences wrapped to (-pi, pi].  Bounds (nuPlan's): longitudinal
    acceleration (|v_t| - |v_{t-1}|) / dt in [-4.05, 2.40] m/s^2 (t >= 2); jerk, its difference / dt, |.| <= 4.13 m/s^3 (t >= 3);
    yaw rate w_t = wrap(psi_t - psi_{t-1}) / dt, |.| <= 0.95 rad/s (t >= 2); yaw acceleration (w_t - w_{t-1}) / dt, |.| <= 1.93
    rad/s^2 (t >= 3); lateral acceleration |v_t| w_t, |.| <= 4.89 m/s^2 (t >= 2).  C = 1 when every term stays within its bound.
  Score.  PDMS = NC x DAC x (5 TTC + 5 EP + 2 C) / 12, NAVSIM's weights, so a trajectory that passes every term and makes
    full progress scores 1.  A trajectory with an invalid step (a non-finite centre or heading)
    scores 0 and is counted in ``invalid``; its terms are not computed and it is left out of the term rates.
  Per sample and trajectory (ops.driving_score_views): the first at-fault and the first exempt collision (step, actor row,
    class), the first TTC violation (step, row), the first off-road step, the comfort mask with each term's first failing step,
    s and L in fp64, and the first invalid step.
  Host reduction (DrivingScores), for plan and for expert, overall and per recorded command: samples, pdms (the mean over every
    sample, invalid ones counting 0), over the valid samples the nc / dac / ttc / comfort pass rates, the mean ep and each
    comfort term's failure rate, the samples with an at-fault and with an exempt collision, invalid, and step_seconds.  A rate
    over no sample is null.
  Not modelled: reactive agents (the recorded traffic does not respond to the plan), lane and driving-direction compliance,
    static objects other than the recorded actors, smoothing, and lane-based at-fault logic for lateral collisions.

With --det-boxes (``det_boxes=True``) the result also holds ``det_boxes``: the detections scored as boxes, by rotated-box IoU
and by the position, size and heading errors of the detections matched at 2 m.  Per batch: one ops.det_box_eval launch on the
packed peaks and the actor table eval_batch reads, and one copy of its result buffer; no extra model call.  The protocol
(lavb_det_box_eval in include/lav_b200.h states every operation):

  Survivors and ground truth.  Those of eval_batch: the same filters, rank order and window, per class.
  Boxes, in map pixels, fp64.  A detection: centre at its peak pixel, half extents packed rows 2-3 (ww, hh), heading (cos, sin)
    = packed rows 4-5, corners centre + (+-ww (-sin, cos) +- hh (-cos, -sin)), the boxes LAVAgent.visualize draws.  An actor:
    centre at det_centre, half extents (bx, by) * ppm, heading (cos, sin)(ori), the targets detections_to_heatmap writes.  A box
    with an extent not finite and > 0, a non-finite heading or centre, or zero area is degenerate: IoU 0 with every box.
  IoU.  The exact intersection area of the two quadrilaterals (the detection's clipped by the actor's, Sutherland-Hodgman, then
    the shoelace formula), I / (A + B - I).
  IoU match.  Per class and threshold 0.3 / 0.5 / 0.7: the survivors in rank order each take the untaken actor of their class
    with the highest IoU >= the threshold, ties to the lower actor row.
  Errors of the 2 m match (eval_batch's, the same pairs): the IoU of the pair; translation = the pixel distance / ppm; scale =
    1 - the IoU of the two boxes with centres and headings aligned (nuScenes' ASE), from the half extents; heading = min(r, 2 pi -
    r), r = fmod(|atan2(sin, cos) - ori|, 2 pi), in [0, pi]; range = the actor's distance from the ego in metres.
  Host reduction (DetBoxScores), per class: n_gt, n_det, ap_iou[t] = average_precision of the survivors at IoU threshold t
    (det[cls].ap's tie rule), matched = the 2 m matches, recall = matched / n_gt, and over the matches the mean IoU,
    translation_m, scale, heading_rad and flipped_rate (the share with a heading error > pi / 2); the same errors per range band
    of the actor's distance, [0, 10), [10, 20) and [20, 30) m.  Heading means skip a non-finite heading error.  A mean over no
    row, and recall and AP with n_gt = 0, are null.

With --brake --bra-weights PATH (``brake=True, bra_model=...``) the result also holds ``brake``: the agent's brake-or-drive
decision (lav_agent_fast.run_step) against the recorded brake flag bra, and each of its three rules on its own.  The decision is
the verdict of the agent's own kernel (lavb_agent_control, control.AgentController's launch); nothing restates it.  The loader
also reads the brake model's camera images (TemporalBatchLoader ``cameras``).  Per batch: one brake-model call for all
checkpoints, then per checkpoint two ops.agent_control launches and one copy of their (B, 3) int32 result.  The protocol:

  Brake model.  agent.brake_model's private copy of bra_model at ``precision`` (the agent's), called through agent.brake_probs
    on the batch's camera bytes: the three middle cameras of camera_yaws side by side and tel_rgb[:-crop_tel_bottom], decoded by
    datasets.load_img (what datasets.CameraDataset reads for evaluate_rgb).  One call per batch, shared by every checkpoint.
  Controls.  ops.agent_control on forward_batch's ego_plan_locs and ego_cast_locs (commands 4 and 5 take the cast in the kernel,
    as in the agent), the brake probabilities, the recorded commands, speeds of 0 and a freshly zeroed controller state per
    launch; the agent's YAML (``agent_config``, --agent-config; default the dataset's config) gives the CONTROLLER keys,
    cmd_thresh and pixels_per_meter (control.control_config).  Rows of the first launch: forward_batch's other_cast_locs /
    other_cast_cmds, the forecasts the agent makes for the vehicles it detects.  Rows of the second (expert_track_rows): the
    recorded futures of the sample's tracked vehicles, label slots 1 <= a < num_objs with typ 1, branch 0 = locs[f, a, 1:] -
    ego_locs[f, 0] (the ego frame of other_cast_locs, as in the --forecast-detected protocol) with score 1, every other branch
    NaN with score 0, so it never collides; built on the device from the batch's label tensors.  The labels are capped at
    max_objs, and pedestrians are not rows: the agent forecasts vehicles only.
  Speed.  Speed enters only the throttle, the speed cap and the creep, none of which is scored; with speed 0 and a fresh state
    the stop counter is 1, far below the 600 ticks that start the creep, so the brake output is exactly the three rules.
  Verdicts per sample.  agent: the control's brake output is 1; brake_model: LAVB_CTL_BRAKE_MODEL (pred_bra > 0.1); plan_stop:
    LAVB_CTL_PID_BRAKE (pid_control's desired speed below brake_speed * ppm; never set on a plan with a NaN, which skips the PID
    step); collide: LAVB_CTL_COLLIDE of the first launch (plan_collide on the detected vehicles' forecasts); collide_expert_tracks:
    LAVB_CTL_COLLIDE of the second (the collision rule with perfect detection and forecasts: its difference from collide is the
    perception and forecast error, not the rule).
  Host reduction (BrakeScores), against the recorded bra (positive when non-zero): per verdict tp, fp, fn, tn, precision =
    tp / (tp + fp), recall = tp / (tp + fn), false_brake_rate = fp / (fp + tn) (the agent brakes, the expert drives: phantom
    braking), missed_brake_rate = fn / (tp + fn) (the expert brakes, the agent drives on); the same per recorded command, for
    every command 0 .. C - 1 the planner has; samples, positives, invalid_plans (LAVB_CTL_PLAN_INVALID); by_reason: for every
    combination of the three rules that fired alone together (brake_model, plan_stop, collide, their pairs and all three) the
    agent brakes it triggered and how many of them were false.  A rate over no sample is null.
  Not scored: the throttle, the steer, the speed cap and the creep (they depend on the speed, which the recording holds only as
    the expert's).

With --seg-weights PATH (``seg_model=...``) the LiDAR rows are painted online by that RGBSegmentationModel, as the agent paints
each sweep when it arrives, instead of read from the recording's lidar_sem keys, which are then never read: a recording that was
never painted can be scored, two segmentation checkpoints can be scored side by side, and the effect of the painting on every
score above can be seen.  The model is loaded strictly, as data_paint and evaluate_paint load it, and runs at ``precision``.
Per batch: the batch's distinct frames decoded once each on the loader's threads, one forward_features_nhwc call over their
images (shared by every checkpoint of a sweep) and one ops.lidar_batch_paint launch in place of ops.lidar_batch.  The result
gains painting = {frames: F, images: 3F}, F the frames segmented over the recording.  The protocol:

  What is painted.  The sample at frame i stacks the sweeps of frames i, i - 1, ..., i - num_frame_stack (those >= 0); each
    sweep is painted with its own frame's images.  That is what data_paint stored for that frame and what the agent painted
    when that sweep arrived.
  Cameras.  Those of data_paint and evaluate_paint: point_painting.make_converters(camera_x, camera_z) with CAMERA_YAWS (-60,
    0, 60), records rgb_0 .. rgb_2 decoded by datasets.load_img (BGR -> RGB), each 288 x 256.  The config's five camera_yaws
    are not the painting cameras.
  Order of operations.  Each row is painted on its raw, unrotated point, before the rotation jitter and the field-of-view
    re-mask of the stored path, so online painting followed by the batch construction equals data_paint followed by the
    stored path, row for row.
  Errors.  A missing rgb_{c} key, or an image of another size, raises LavbError naming the trajectory and the key, before the
    batch is built.
With --brake the brake model's camera reads are unchanged.
"""
import argparse
import json

import numpy as np
import torch

from . import ops
from .agent import brake_model, brake_probs, infer_model, math_mode
from .capi import LavbError
from .control import FLAG_BRAKE_MODEL, FLAG_COLLIDE, FLAG_PID_BRAKE, FLAG_PLAN_INVALID, control_config
from .datasets import TemporalBatchLoader, TemporalLiDARPaintedDataset
from .eval_sweep import (ResidentMeter, add_checkpoint_args, check_sweep_fits, eval_device, gather_merged, init_ranks,
                         rank_and_world, select_checkpoints, sweep_json, sweep_table)
from .heads import off_centre
from .model_inference import peak_filter

CLASSES = ("pedestrian", "vehicle")


def average_precision(scores, matched, n_gt):
    """all-point-interpolated AP of detections (scores, matched flags) against n_gt ground-truth objects; None when n_gt is 0."""
    if n_gt == 0:
        return None
    order = np.argsort(-np.asarray(scores, np.float64), kind="stable")
    tp = np.cumsum(np.asarray(matched, bool)[order])
    precision = tp / np.arange(1, len(tp) + 1)
    recall = tp / n_gt
    envelope = np.maximum.accumulate(precision[::-1])[::-1]
    return float((envelope * np.diff(np.concatenate([[0.0], recall]))).sum())


class Scores:
    """host accumulation of eval_batch results over a recording."""

    def __init__(self):
        self.iou = np.zeros((3, 2), np.int64)
        self.ngt = np.zeros(2, np.int64)
        self.det = [[] for _ in CLASSES]             # per class: (score, flags) arrays of the surviving detections, in order
        self.ade, self.fde, self.cmd = [], [], []

    def add(self, v, cmds):
        """v = ops.eval_views of a host copy of one batch's result buffer; cmds (B,) the recorded commands."""
        self.iou += v["iou"].numpy().sum(0)
        self.ngt += v["ngt"].numpy().sum(0)
        score, flags = v["score"].numpy(), v["flags"].numpy()
        n_det = score.shape[1] // 2
        for c in range(2):
            s, f = score[:, c * n_det:(c + 1) * n_det], flags[:, c * n_det:(c + 1) * n_det]
            keep = (f & 16) != 0
            self.det[c].append((s[keep], f[keep]))
        pe = v["plan_err"].numpy()
        self.ade += pe[:, 0].tolist()
        self.fde += pe[:, 1].tolist()
        self.cmd += [int(c) for c in cmds]

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order (a later rank's shard)."""
        self.iou += other.iou
        self.ngt += other.ngt
        for c in range(len(CLASSES)):
            self.det[c] += other.det[c]
        self.ade += other.ade
        self.fde += other.fde
        self.cmd += other.cmd

    def summary(self):
        inter, union = self.iou[:, 0], self.iou[:, 1]
        det = {}
        for c, name in enumerate(CLASSES):
            s = np.concatenate([a for a, _ in self.det[c]] or [np.zeros(0, np.float32)])
            f = np.concatenate([b for _, b in self.det[c]] or [np.zeros(0, np.int32)])
            aps = {f"{t:g}": average_precision(s, (f >> k) & 1, int(self.ngt[c])) for k, t in enumerate(ops.EVAL_THRESHOLDS_M)}
            aps["mean"] = None if self.ngt[c] == 0 else float(np.mean(list(aps.values())))
            det[name] = dict(ap=aps, n_gt=int(self.ngt[c]), n_det=int(len(s)))
        ade, fde, cmd = np.array(self.ade), np.array(self.fde), np.array(self.cmd, np.int64)
        plan = dict(ade=float(ade.mean()) if len(ade) else None, fde=float(fde.mean()) if len(fde) else None,
                    per_cmd={str(c): dict(samples=int((cmd == c).sum()), ade=float(ade[cmd == c].mean()), fde=float(fde[cmd == c].mean()))
                             for c in sorted(set(cmd.tolist()))})
        return dict(samples=len(self.ade), bev_iou=[float(i) / float(u) if u else None for i, u in zip(inter, union)],
                    bev_counts=self.iou.tolist(), det=det, plan=plan)


FORECAST_MISS_M = 2.0       # a vehicle row whose minFDE exceeds this counts as a miss


def score_forecasts(fc, cmds, plan=False):
    """one ops.forecast_eval launch over a forecast_recorded result: its K vehicle rows (no command), its B ego casts and, with
    ``plan``, its B ego plans (those two under the recorded commands ``cmds``, a (B,) device tensor).  -> the result buffer."""
    K = fc["cast"].shape[0]
    parts = [(fc["cast"], fc["score"], fc["target"]), (fc["ego_cast"], fc["ego_score"], fc["ego_target"])]
    if plan:
        parts.append((fc["ego_plan"], fc["ego_score"], fc["ego_target"]))
    cat = lambda i: torch.cat([p[i].float() for p in parts]).contiguous()
    cmd = torch.cat([torch.full((K,), -1, dtype=torch.int32, device=cmds.device)] + [cmds.to(torch.int32)] * (len(parts) - 1))
    return ops.forecast_eval(cat(0), cat(1), cat(2), cmd)


class ForecastScores:
    """host accumulation of score_forecasts results over a recording."""

    def __init__(self, plan=False):
        self.plan = plan
        self.other, self.ego, self.top, self.ego_plan, self.cmd = [], [], [], [], []

    def add(self, v, n_other, cmds):
        """v = ops.forecast_views of a host copy of one batch's result buffer; n_other its vehicle rows; cmds (B,) the recorded
        commands, on the host."""
        err, branch = v["err"].numpy(), v["branch"].numpy()
        b = len(cmds)
        self.other.append(err[:n_other])
        self.ego.append(err[n_other:n_other + b])
        self.top.append(branch[n_other:n_other + b, 1])
        if self.plan:
            self.ego_plan.append(err[n_other + b:n_other + 2 * b])
        self.cmd.append(np.asarray(cmds, np.int64))

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order."""
        for k in ("other", "ego", "top", "ego_plan", "cmd"):
            getattr(self, k).extend(getattr(other, k))

    def summary(self):
        mean = lambda a: float(np.mean(a)) if len(a) else None
        rows = lambda parts: np.concatenate(parts) if parts else np.zeros((0, 6))
        o, e, cmd = rows(self.other), rows(self.ego), np.concatenate(self.cmd) if self.cmd else np.zeros(0, np.int64)
        top = np.concatenate(self.top) if self.top else np.zeros(0, np.int32)

        def ego(m):
            return dict(samples=int(m.sum()), ade=mean(e[m, 4]), fde=mean(e[m, 5]), min_ade=mean(e[m, 0]), min_fde=mean(e[m, 1]),
                        cmd_accuracy=mean(top[m] == cmd[m]))
        cmds, every = sorted(set(cmd.tolist())), np.ones(len(cmd), bool)
        r = dict(other=dict(rows=len(o), min_ade=mean(o[:, 0]), min_fde=mean(o[:, 1]), top_ade=mean(o[:, 2]), top_fde=mean(o[:, 3]),
                            miss_rate=mean(o[:, 1] > FORECAST_MISS_M)),
                 ego_cast=dict(ego(every), per_cmd={str(c): ego(cmd == c) for c in cmds}))
        if self.plan:
            p = rows(self.ego_plan)
            plan = lambda m: dict(samples=int(m.sum()), ade=mean(p[m, 4]), fde=mean(p[m, 5]))
            r["ego_plan"] = dict(plan(every), per_cmd={str(c): plan(cmd == c) for c in cmds})
        return r


def format_forecast(f):
    """the printout lines of a ForecastScores summary."""
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    o, e = f["other"], f["ego_cast"]
    lines = [f"forecast, other vehicles ({o['rows']} rows): minADE {fmt(o['min_ade'])} m, minFDE {fmt(o['min_fde'])} m, "
             f"top-1 ADE {fmt(o['top_ade'])} m, FDE {fmt(o['top_fde'])} m, miss rate {fmt(o['miss_rate'])}",
             f"forecast, ego cast: ADE {fmt(e['ade'])} m, FDE {fmt(e['fde'])} m, minADE {fmt(e['min_ade'])} m, "
             f"minFDE {fmt(e['min_fde'])} m, command accuracy {fmt(e['cmd_accuracy'])}"]
    lines += [f"  cmd {c}: {d['samples']} samples, ADE {fmt(d['ade'])} m, FDE {fmt(d['fde'])} m, minADE {fmt(d['min_ade'])} m, "
              f"minFDE {fmt(d['min_fde'])} m, accuracy {fmt(d['cmd_accuracy'])}" for c, d in e["per_cmd"].items()]
    if "ego_plan" in f:
        p = f["ego_plan"]
        lines.append(f"ego plan: ADE {fmt(p['ade'])} m, FDE {fmt(p['fde'])} m")
        lines += [f"  cmd {c}: {d['samples']} samples, ADE {fmt(d['ade'])} m, FDE {fmt(d['fde'])} m" for c, d in p["per_cmd"].items()]
    return lines


def detected_rows(packed, pixels_per_meter, centre, min_score=0.2):
    """The row table of the forecasts on detected vehicles: the class-1 peaks of host ``packed`` (B, 7, 2 * n_det) that
    decode_packed keeps and det_to_locs forecasts (``centre`` = UniPlanner.crop_centre), in frame, then column order.  -> dict:
    frame (K,) int64, col (K,) int32 = the packed column, score (K,) fp32, locs (K, 2) fp32 = det_to_locs' ego metres, counts (B,)."""
    keep, x, y, cls = peak_filter(packed, pixels_per_meter, 2, min_score)
    keep = keep & (cls[None] == 1) & off_centre(x, y, *centre)
    frame, col = np.nonzero(keep)
    X, Y = x[frame, col], y[frame, col]
    locs = np.stack([(X - centre[0]) / pixels_per_meter, (Y - centre[1]) / pixels_per_meter], 1).astype(np.float32).reshape(-1, 2)
    return dict(frame=frame, col=col.astype(np.int32), score=packed[frame, 0, col].astype(np.float32), locs=locs,
                counts=keep.sum(1))


def score_detected(out, rows, actors, offsets, locs, ego_locs, num_objs, grid):
    """one ops.det_forecast_match launch and one ops.forecast_eval launch into its buffer: forward_batch's output ``out``, its
    detected_rows ``rows``, eval_batch's actor table and the labels locs / ego_locs / num_objs (host).  -> the result buffer."""
    counts = [len(c) for c in out["other_cast_locs"]]
    if rows["counts"].tolist() != counts:
        raise LavbError(f"forecast rows per frame {rows['counts'].tolist()} differ from the forecasts infer_batch made {counts}")
    b, k = len(counts), len(rows["col"])
    row_offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    buf = ops.det_forecast_match(out["packed"], actors, offsets, row_offsets, rows["col"], num_objs, locs, ego_locs, grid)
    cast = torch.cat(out["other_cast_locs"]).float().contiguous()
    score = torch.cat(out["other_cast_cmds"]).float().contiguous()
    target = ops.det_match_views(buf, b, k, locs.shape[2] - 1)["target"]
    ops.forecast_eval(cast, score, target, torch.full((k,), -1, dtype=torch.int32, device=cast.device), out=buf[:56 * k])
    return buf


class DetectedForecastScores:
    """host accumulation of score_detected results over a recording."""

    def __init__(self, match_m=ops.DET_MATCH_M):
        self.match_m = match_m
        self.score, self.flag, self.err = [], [], []
        self.gt = 0

    def add(self, v, scores):
        """v = ops.det_match_views of a host copy of one batch's result buffer; scores (K,) the rows' detection scores."""
        self.score.append(np.asarray(scores, np.float32))
        self.flag.append(v["flag"].numpy().copy())
        self.err.append(v["err"].numpy()[:, :4].copy())
        self.gt += int(v["ngt"].numpy()[:, 0].sum())

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order."""
        self.score += other.score
        self.flag += other.flag
        self.err += other.err
        self.gt += other.gt

    def summary(self):
        mean = lambda a: float(np.mean(a)) if len(a) else None
        s = np.concatenate(self.score) if self.score else np.zeros(0, np.float32)
        f = np.concatenate(self.flag) if self.flag else np.zeros(0, np.int32)
        e = np.concatenate(self.err) if self.err else np.zeros((0, 4))
        tracked, untracked = (f & 2) != 0, ((f & 1) != 0) & ((f & 2) == 0)
        m = e[tracked]
        tp = tracked & (e[:, 1] <= FORECAST_MISS_M)
        n = int(tracked.sum())
        return dict(rows=len(f), matched=n, matched_untracked=int(untracked.sum()), gt=self.gt,
                    recall=n / self.gt if self.gt else None, min_ade=mean(m[:, 0]), min_fde=mean(m[:, 1]), top_ade=mean(m[:, 2]),
                    top_fde=mean(m[:, 3]), miss_rate=mean(m[:, 1] > FORECAST_MISS_M),
                    ap=average_precision(s[~untracked], tp[~untracked], self.gt), match_m=self.match_m)


DET_BOX_RANGES_M = ((0, 10), (10, 20), (20, 30))      # range bands of the box errors, by the matched actor's distance


class DetBoxScores:
    """host accumulation of ops.det_box_eval results over a recording."""

    def __init__(self):
        self.score, self.flags, self.err = [[] for _ in CLASSES], [[] for _ in CLASSES], [[] for _ in CLASSES]
        self.ngt = np.zeros(len(CLASSES), np.int64)

    def add(self, v):
        """v = ops.det_box_views of a host copy of one batch's result buffer."""
        score, flags, err = v["score"].numpy(), v["flags"].numpy(), v["err"].numpy()
        n_det = score.shape[1] // 2
        for c in range(len(CLASSES)):
            s, f, e = (a[:, c * n_det:(c + 1) * n_det] for a in (score, flags, err))
            keep = (f & 16) != 0
            self.score[c].append(s[keep].copy())
            self.flags[c].append(f[keep].copy())
            self.err[c].append(e[keep].copy())
        self.ngt += v["ngt"].numpy().sum(0)

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order."""
        for c in range(len(CLASSES)):
            self.score[c] += other.score[c]
            self.flags[c] += other.flags[c]
            self.err[c] += other.err[c]
        self.ngt += other.ngt

    @staticmethod
    def errors(e):
        """the means over the matched rows ``e`` (k, 5) of ops.DET_BOX_ERRORS; the heading's over its finite values."""
        mean = lambda a: float(np.mean(a)) if len(a) else None
        h = e[:, 3][np.isfinite(e[:, 3])]
        return dict(matched=len(e), mean_iou=mean(e[:, 0]), translation_m=mean(e[:, 1]), scale=mean(e[:, 2]), heading_rad=mean(h),
                    flipped_rate=mean(h > np.pi / 2))

    def summary(self):
        out = {}
        for c, name in enumerate(CLASSES):
            s = np.concatenate(self.score[c]) if self.score[c] else np.zeros(0, np.float32)
            f = np.concatenate(self.flags[c]) if self.flags[c] else np.zeros(0, np.int32)
            e = np.concatenate(self.err[c]) if self.err[c] else np.zeros((0, len(ops.DET_BOX_ERRORS)))
            n_gt = int(self.ngt[c])
            m = e[(f & 8) != 0]
            d = dict(n_gt=n_gt, n_det=len(s),
                     ap_iou={f"{t:g}": average_precision(s, (f >> k) & 1, n_gt) for k, t in enumerate(ops.DET_BOX_IOU_THRESHOLDS)},
                     recall=len(m) / n_gt if n_gt else None, **self.errors(m))
            d["by_range"] = {f"{lo}-{hi}": self.errors(m[(m[:, 4] >= lo) & (m[:, 4] < hi)]) for lo, hi in DET_BOX_RANGES_M}
            out[name] = d
        return out


def format_det_boxes(r):
    """the printout lines of a DetBoxScores summary."""
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    errs = lambda d: (f"IoU {fmt(d['mean_iou'])}, translation {fmt(d['translation_m'])} m, scale {fmt(d['scale'])}, heading "
                      f"{fmt(d['heading_rad'])} rad, flipped {fmt(d['flipped_rate'])}")
    lines = []
    for name, d in r.items():
        lines.append(f"det boxes, {name} ({d['n_gt']} GT, {d['n_det']} detections): AP at IoU " +
                     " ".join(f"{k}={fmt(v)}" for k, v in d["ap_iou"].items()) +
                     f"; {d['matched']} matched at 2 m, recall {fmt(d['recall'])}: " + errs(d))
        lines += [f"  {band} m: {e['matched']} matched, " + errs(e) for band, e in d["by_range"].items()]
    return lines


PLAN_SAFETY_TRAJECTORIES = ("plan", "expert")
DRIVING_SCORE_WEIGHTS = (5.0, 5.0, 2.0)      # TTC, EP and C in the PDMS (NAVSIM's), over their sum 12
DRIVING_SCORE_MIN_LENGTH_M = 5.0             # an expert shorter than this gives EP 1


def score_plan_safety(plan, ego_locs, table, bev, grid):
    """one ops.plan_safety launch over a batch's ego plans ``plan`` (B,T,2) and experts ego_locs[:, 1:], against the batch's
    packed plan_safety tables (stage_plan_safety, on the host) and the road plane of its ``bev``.  -> (B, 2, 8) int32 on the
    device, trajectory 0 the plan, 1 the expert."""
    dev = bev.device
    traj = torch.stack([plan.float(), ego_locs[:, 1:].float()], 1).contiguous()
    return ops.plan_safety(traj, table["actors"].to(dev, non_blocking=True), table["offsets"],
                           table["ego_ext"].to(dev, non_blocking=True), bev, grid)


class PlanSafetyScores:
    """host accumulation of score_plan_safety results over a recording."""

    def __init__(self, names=PLAN_SAFETY_TRAJECTORIES):
        self.names = names
        self.res, self.cmd = [], []

    def add(self, res, cmds):
        """res (B, n, 8) int32, a host copy of one batch's result; cmds (B,) the recorded commands."""
        self.res.append(np.asarray(res, np.int32).copy())
        self.cmd.append(np.asarray(cmds, np.int64))

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order."""
        self.res += other.res
        self.cmd += other.cmd

    def summary(self, t):
        """per trajectory: the rates over all samples and per recorded command (``t`` steps per trajectory)."""
        res = np.concatenate(self.res) if self.res else np.zeros((0, len(self.names), 8), np.int32)
        cmd = np.concatenate(self.cmd) if self.cmd else np.zeros(0, np.int64)

        def rates(r):
            n = len(r)
            rate = lambda hit: float(hit.mean()) if n else None
            first = r[:, 7]
            return dict(samples=n, collision_rate=rate(first > 0), vehicle_collision_rate=rate(r[:, 0] > 0),
                        pedestrian_collision_rate=rate(r[:, 2] > 0), off_road_rate=rate(r[:, 4] > 0),
                        collision_rate_by_step=[rate((first > 0) & (first <= s)) for s in range(1, t + 1)],
                        off_map_steps=int(r[:, 5].sum()), invalid_steps=int(r[:, 6].sum()))

        out = {}
        for j, name in enumerate(self.names):
            r = res[:, j]
            out[name] = dict(rates(r), per_cmd={str(c): rates(r[cmd == c]) for c in sorted(set(cmd.tolist()))})
        return out


def score_driving(plan, ego_locs, table, bev, grid, dt=ops.DRIVING_SCORE_STEP_S):
    """one ops.driving_score launch over a batch's ego plans ``plan`` (B,T,2) and experts ego_locs[:, 1:], against the batch's
    packed driving_score tables (stage_plan_safety, on the host) and the road plane of its ``bev``, at step period ``dt``.  -> the
    result buffer on the device (ops.driving_score_views with n = 2), trajectory 0 the plan, 1 the expert."""
    dev = bev.device
    expert = ego_locs[:, 1:].float().contiguous()
    traj = torch.stack([plan.float(), expert], 1).contiguous()
    return ops.driving_score(traj, expert, table["actors"].to(dev, non_blocking=True), table["offsets"],
                             table["ego_ext"].to(dev, non_blocking=True), bev, grid, dt)


def driving_terms(v):
    """the per-trajectory terms of driving_score_views ``v`` (numpy arrays): dict of invalid, nc, dac, ttc, comfort, at_fault,
    exempt (bool), ep and pdms (fp64), and comfort_fail (..., 5) bool, one entry per ops.DRIVING_SCORE_COMFORT term."""
    invalid = v["invalid_step"] > 0
    nc, dac, ttc = v["fault_step"] < 0, v["off_road_step"] < 0, v["ttc_step"] < 0
    mask = v["comfort_mask"]
    comfort = mask == 0
    s, length = v["progress"], v["length"]
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = s / length
        ep = np.where(length < DRIVING_SCORE_MIN_LENGTH_M, 1.0, np.where(np.isnan(ratio), 0.0, np.clip(ratio, 0.0, 1.0)))
    w_ttc, w_ep, w_c = DRIVING_SCORE_WEIGHTS
    pdms = np.where(invalid, 0.0, nc * dac * (w_ttc * ttc + w_ep * ep + w_c * comfort) / (w_ttc + w_ep + w_c))
    fail = np.stack([(mask >> q) & 1 for q in range(len(ops.DRIVING_SCORE_COMFORT))], -1) != 0
    return dict(invalid=invalid, nc=nc, dac=dac, ttc=ttc, comfort=comfort, at_fault=~nc, exempt=v["exempt_step"] > 0, ep=ep,
                pdms=pdms, comfort_fail=fail)


class DrivingScores:
    """host accumulation of score_driving results over a recording."""

    def __init__(self, names=PLAN_SAFETY_TRAJECTORIES, dt=ops.DRIVING_SCORE_STEP_S):
        self.names, self.dt = names, dt
        self.res, self.ep, self.cmd = [], [], []

    def add(self, buf, cmds):
        """buf = a host copy of one batch's result buffer; cmds (B,) the recorded commands."""
        b = len(cmds)
        v = ops.driving_score_views(buf, b, len(self.names))
        self.res.append(torch.stack([v[k] for k in ops.DRIVING_SCORE_FIELDS], -1).numpy().copy())
        self.ep.append(torch.stack([v["progress"], v["length"]], -1).numpy().copy())
        self.cmd.append(np.asarray(cmds, np.int64).reshape(-1))

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order."""
        self.res += other.res
        self.ep += other.ep
        self.cmd += other.cmd

    def terms(self):
        """driving_terms of every record, (samples, trajectories) each, and the recorded commands."""
        n, f = len(self.names), len(ops.DRIVING_SCORE_FIELDS)
        res = np.concatenate(self.res) if self.res else np.zeros((0, n, f), np.int32)
        ep = np.concatenate(self.ep) if self.ep else np.zeros((0, n, 2))
        v = {k: res[..., i] for i, k in enumerate(ops.DRIVING_SCORE_FIELDS)}
        v["progress"], v["length"] = ep[..., 0], ep[..., 1]
        return driving_terms(v), np.concatenate(self.cmd) if self.cmd else np.zeros(0, np.int64)

    def summary(self):
        """per trajectory: the score and its terms over all samples and per recorded command."""
        d, cmd = self.terms()

        def stats(m, j):
            mean = lambda a: float(np.mean(a)) if len(a) else None
            ok = m & ~d["invalid"][:, j]
            fail = d["comfort_fail"][ok, j]
            return dict(samples=int(m.sum()), pdms=mean(d["pdms"][m, j]), nc=mean(d["nc"][ok, j]), dac=mean(d["dac"][ok, j]),
                        ttc=mean(d["ttc"][ok, j]), comfort=mean(d["comfort"][ok, j]), ep=mean(d["ep"][ok, j]),
                        comfort_failure_rate={name: mean(fail[:, q]) for q, name in enumerate(ops.DRIVING_SCORE_COMFORT)},
                        at_fault_collisions=int(d["at_fault"][ok, j].sum()), exempt_collisions=int(d["exempt"][ok, j].sum()),
                        invalid=int(d["invalid"][m, j].sum()))

        out = {}
        every = np.ones(len(cmd), bool)
        for j, name in enumerate(self.names):
            out[name] = dict(stats(every, j), per_cmd={str(c): stats(cmd == c, j) for c in sorted(set(cmd.tolist()))})
        out["step_seconds"] = self.dt
        return out


def format_driving_score(s):
    """the printout lines of a DrivingScores summary."""
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    line = lambda d: (f"{d['samples']} samples, PDMS {fmt(d['pdms'])}: NC {fmt(d['nc'])}, DAC {fmt(d['dac'])}, TTC {fmt(d['ttc'])}, "
                      f"EP {fmt(d['ep'])}, comfort {fmt(d['comfort'])}; {d['at_fault_collisions']} at-fault and "
                      f"{d['exempt_collisions']} exempt collisions, {d['invalid']} invalid")
    lines = []
    for name in (k for k in s if k != "step_seconds"):
        d = s[name]
        lines.append(f"driving score, {name} (dt {s['step_seconds']:g} s): " + line(d))
        lines.append("  comfort failures: " + ", ".join(f"{k} {fmt(v)}" for k, v in d["comfort_failure_rate"].items()))
        lines += [f"  cmd {c}: " + line(e) for c, e in d["per_cmd"].items()]
    return lines


def format_plan_safety(s):
    """the printout lines of a PlanSafetyScores summary."""
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    line = lambda d: (f"{d['samples']} samples, collision rate {fmt(d['collision_rate'])} (vehicles "
                      f"{fmt(d['vehicle_collision_rate'])}, pedestrians {fmt(d['pedestrian_collision_rate'])}), off-road rate "
                      f"{fmt(d['off_road_rate'])}, {d['off_map_steps']} off-map steps, {d['invalid_steps']} invalid steps")
    lines = []
    for name, d in s.items():
        lines.append(f"plan safety, {name}: " + line(d))
        lines += [f"  cmd {c}: " + line(e) for c, e in d["per_cmd"].items()]
    return lines


BRAKE_VERDICTS = ("agent", "brake_model", "plan_stop", "collide", "collide_expert_tracks")
BRAKE_REASONS = (("brake_model", FLAG_BRAKE_MODEL), ("plan_stop", FLAG_PID_BRAKE), ("collide", FLAG_COLLIDE))


def expert_track_rows(locs, ego_locs, typs, num_objs, num_cmds):
    """The recorded futures of a batch's tracked vehicles as forecast rows of ops.agent_control, built on the device of the label
    tensors locs (B, M, T+1, 2), ego_locs (B, T+1, 2) and typs (B, M) from num_objs (B,) with no host loop.  Every label slot
    1 .. M - 1 of a sample is a row, sample b owning rows [b (M - 1), (b + 1)(M - 1)); a slot a < num_objs[b] with typs[b, a] ==
    1 has branch 0 = locs[b, a, 1:] - ego_locs[b, 0] with score 1, and every other branch, and every branch of any other slot,
    NaN points with score 0, which never collide.  -> (rows (B (M - 1), num_cmds, T, 2) fp32, scores (B (M - 1), num_cmds) fp32,
    offsets (B + 1,) int32 on the host)."""
    B, M = typs.shape
    dev = locs.device
    n = torch.as_tensor(num_objs).to(dev).reshape(B, 1)
    live = (typs[:, 1:] == 1) & (torch.arange(1, M, device=dev)[None] < n)                   # (B, M - 1)
    track = (locs[:, 1:, 1:] - ego_locs[:, None, :1]).float()                                  # (B, M - 1, T, 2)
    T = track.shape[2]
    rows = torch.full((B, M - 1, num_cmds, T, 2), float("nan"), device=dev)
    rows[:, :, 0] = torch.where(live[..., None, None], track, rows[:, :, 0])
    scores = torch.zeros((B, M - 1, num_cmds), device=dev)
    scores[:, :, 0] = live.float()
    return rows.reshape(-1, num_cmds, T, 2), scores.reshape(-1, num_cmds), np.arange(B + 1, dtype=np.int32) * (M - 1)


def score_brake(out, pred_bra, expert, cmds, config):
    """The agent's brake decision on one batch: two ops.agent_control launches on forward_batch's ``out`` and the brake
    probabilities ``pred_bra`` (B,), each from a freshly zeroed controller state, with speeds 0 and the recorded commands
    ``cmds`` (B,) on the host; the first with the detected vehicles' forecasts as rows, the second with ``expert`` (the
    expert_track_rows triple).  ``config`` is a capi.ControlConfig.  -> (B, 3) int32 on the device: the flags, the flags on the
    recorded tracks, and the agent's brake (control[:, 2] == 1)."""
    plan, cast = out["ego_plan_locs"].float().contiguous(), out["ego_cast_locs"].float().contiguous()
    B, dev = plan.shape[0], plan.device
    offsets = np.concatenate([[0], np.cumsum([len(o) for o in out["other_cast_locs"]])]).astype(np.int32)
    detected = (torch.cat(list(out["other_cast_locs"])).float().contiguous(),
                torch.cat(list(out["other_cast_cmds"])).float().contiguous(), offsets)
    speed = torch.zeros(B, device=dev)
    pred = pred_bra.reshape(B).float().contiguous()
    record = ops.agent_control_state_bytes(config.turn_n, config.speed_n)
    controls, flags = [], []
    for rows, scores, offs in (detected, expert):
        state = torch.zeros(B * record, dtype=torch.uint8, device=dev)
        control, f = ops.agent_control(plan, cast, rows, scores, offs, pred, speed, cmds, config, state)
        controls.append(control)
        flags.append(f)
    return torch.stack([flags[0], flags[1], (controls[0][:, 2] == 1).to(torch.int32)], 1)


def brake_verdicts(res):
    """the (n, 5) bool verdicts of BRAKE_VERDICTS of score_brake results ``res`` (n, 3) on the host."""
    res = np.asarray(res).reshape(-1, 3)
    f, fe = res[:, 0], res[:, 1]
    return np.stack([res[:, 2] != 0, (f & FLAG_BRAKE_MODEL) != 0, (f & FLAG_PID_BRAKE) != 0, (f & FLAG_COLLIDE) != 0,
                     (fe & FLAG_COLLIDE) != 0], 1)


def brake_table(fire, y):
    """the counts and rates of brake verdicts ``fire`` (n,) against the recorded brakes ``y`` (n,), both bool."""
    tp, fp = int((fire & y).sum()), int((fire & ~y).sum())
    fn, tn = int((~fire & y).sum()), int((~fire & ~y).sum())
    div = lambda a, b: a / b if b else None
    return dict(tp=tp, fp=fp, fn=fn, tn=tn, precision=div(tp, tp + fp), recall=div(tp, tp + fn), false_brake_rate=div(fp, fp + tn),
                missed_brake_rate=div(fn, tp + fn))


class BrakeScores:
    """host accumulation of score_brake results over a recording, for a planner of ``num_cmds`` command branches."""

    def __init__(self, num_cmds=6):
        self.num_cmds = num_cmds
        self.res, self.cmd, self.bra = [], [], []

    def add(self, res, cmds, bras):
        """res (B, 3) int32, a host copy of one batch's score_brake result; cmds (B,) the recorded commands; bras (B,) the
        recorded brake flags."""
        self.res.append(np.asarray(res, np.int32).reshape(-1, 3).copy())
        self.cmd.append(np.asarray(cmds, np.int64).reshape(-1))
        self.bra.append(np.asarray(bras, np.int64).reshape(-1))

    def extend(self, other):
        """append the records of ``other``, which follow this one's in sample order."""
        self.res += other.res
        self.cmd += other.cmd
        self.bra += other.bra

    def summary(self):
        res = np.concatenate(self.res) if self.res else np.zeros((0, 3), np.int32)
        cmd = np.concatenate(self.cmd) if self.cmd else np.zeros(0, np.int64)
        y = (np.concatenate(self.bra) if self.bra else np.zeros(0, np.int64)) != 0
        v = brake_verdicts(res)
        tables = lambda m: {name: brake_table(v[m, j], y[m]) for j, name in enumerate(BRAKE_VERDICTS)}
        cmds = sorted(set(range(self.num_cmds)) | set(cmd.tolist()))
        agent = v[:, 0]
        fired = np.stack([(res[:, 0] & bit) != 0 for _, bit in BRAKE_REASONS], 1)
        by_reason = {}
        for mask in range(1, 1 << len(BRAKE_REASONS)):
            want = np.array([(mask >> k) & 1 for k in range(len(BRAKE_REASONS))], bool)
            hit = agent & (fired == want[None]).all(1)
            by_reason["+".join(n for (n, _), w in zip(BRAKE_REASONS, want) if w)] = dict(brakes=int(hit.sum()),
                                                                                          false_brakes=int((hit & ~y).sum()))
        return dict(samples=len(res), positives=int(y.sum()), invalid_plans=int(((res[:, 0] & FLAG_PLAN_INVALID) != 0).sum()),
                    verdicts=tables(np.ones(len(res), bool)), per_cmd={str(c): dict(samples=int((cmd == c).sum()), verdicts=tables(cmd == c))
                                                                      for c in cmds},
                    by_reason=by_reason)


def format_brake(b):
    """the printout lines of a BrakeScores summary."""
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    line = lambda d: (f"tp {d['tp']} fp {d['fp']} fn {d['fn']} tn {d['tn']}, precision {fmt(d['precision'])}, recall "
                      f"{fmt(d['recall'])}, false brake rate {fmt(d['false_brake_rate'])}, missed brake rate "
                      f"{fmt(d['missed_brake_rate'])}")
    lines = [f"brake decision ({b['samples']} samples, {b['positives']} recorded brakes, {b['invalid_plans']} invalid plans):"]
    lines += [f"  {name}: " + line(d) for name, d in b["verdicts"].items()]
    lines += [f"  cmd {c} ({d['samples']} samples), agent: " + line(d["verdicts"]["agent"]) for c, d in b["per_cmd"].items()]
    lines.append("  agent brakes by the rules that fired: " +
                 ", ".join(f"{k} {d['brakes']} ({d['false_brakes']} false)" for k, d in b["by_reason"].items()))
    return lines


class PaintingCount:
    """the frames segmented for online painting over a recording."""

    def __init__(self):
        self.frames = 0

    def extend(self, other):
        self.frames += other.frames

    def summary(self, ncam=3):
        return dict(frames=self.frames, images=ncam * self.frames)


def evaluate(lidar_model, uniplanner, dataset, batch_size=32, precision="f16", num_workers=16, forecast=False,
             forecast_detected=False, plan_safety=False, det_boxes=False, brake=False, bra_model=None, agent_config=None,
             seg_model=None, driving_score=False, step_seconds=ops.DRIVING_SCORE_STEP_S):
    """Scores of ``lidar_model`` and ``uniplanner`` over every sample of ``dataset`` (a TemporalLiDARPaintedDataset), the models
    run as the agent runs them at ``precision``; with ``forecast`` also the UniPlanner's forecast scores on the recorded poses,
    with ``forecast_detected`` those on the detected vehicles, with ``plan_safety`` the collision and off-road rates of the ego
    plan and of the expert, with ``det_boxes`` the detections' box scores, with ``brake`` the agent's brake decision with the
    brake model ``bra_model`` under the controls of ``agent_config`` (the agent's YAML dict; default the dataset's config); with
    ``seg_model`` (an RGBSegmentationModel) the sweeps painted online by it instead of read from lidar_sem; with ``driving_score``
    the driving score of the ego plan and of the expert at a step period of ``step_seconds``.
    -> dict (see the module docstring); None on a rank other than 0 of a process group."""
    results = evaluate_checkpoints([(lidar_model, uniplanner)], dataset, batch_size, precision, num_workers, forecast,
                                   forecast_detected, plan_safety, det_boxes, brake, bra_model, agent_config, seg_model,
                                   driving_score, step_seconds)
    return None if results is None else results[0]


@torch.no_grad()
def evaluate_checkpoints(pairs, dataset, batch_size=32, precision="f16", num_workers=16, forecast=False, forecast_detected=False,
                         plan_safety=False, det_boxes=False, brake=False, bra_model=None, agent_config=None, seg_model=None,
                         driving_score=False, step_seconds=ops.DRIVING_SCORE_STEP_S):
    """evaluate() of every (lidar_model, uniplanner) of ``pairs`` in one pass over ``dataset``: each batch is loaded and staged
    once, then every pair runs its own InferModel and scoring launches on it into its own accumulators.  All pairs stay
    resident; a sweep that would not fit on the device is refused before any data is loaded.  With ``brake`` the one brake
    model ``bra_model`` is resident once, before the pairs are measured, and runs once per batch for all pairs; so is the
    segmentation model ``seg_model``, whose painting of each batch all pairs share.  In a process
    group each rank scores its contiguous shard of the recording and rank 0 merges the ranks' records
    (eval_sweep.gather_merged).  -> one evaluate() result per pair on rank 0, None on the other ranks."""
    dev = dataset.device
    rank, world = rank_and_world()
    bra = ctl = None
    if brake:
        if bra_model is None or not pairs:
            raise LavbError("evaluate: brake=True needs the brake model (bra_model) and a checkpoint")
        num_cmds = pairs[0][1].num_cmds
        agent_config = dataset.cfg if agent_config is None else agent_config
        aim = agent_config.get("aim_point")
        if not isinstance(aim, (list, tuple)) or len(aim) != num_cmds:       # config_v2.yaml's aim_point is the trainer's scalar
            raise LavbError(f"evaluate: brake needs the agent's config, whose aim_point has one entry per command of the planner "
                            f"({num_cmds}); this one has {aim!r} (--agent-config)")
        ctl = control_config(agent_config)
        bra = brake_model(bra_model.to(dev).eval(), precision)
    if seg_model is not None:
        n_cls = seg_model.erfnet.decoder.output_conv.out_channels
        if n_cls != len(dataset.seg_channels) + 1:
            raise LavbError(f"evaluate: the seg model has {n_cls} classes, seg_channels gives {len(dataset.seg_channels) + 1}")
        seg_model.to(dev).eval().set_precision(precision)
    models = []
    for i, (lid, uni) in enumerate(pairs):
        meter = ResidentMeter(dev, lid, uni) if i == 0 and len(pairs) > 1 else None
        lid.to(dev).eval()
        uni.to(dev).eval()
        models.append(infer_model(lid, uni, precision, dataset.camera_x, dataset.camera_z, dev))
        if meter is not None:
            check_sweep_fits(len(pairs), meter.resident(), meter.available, batch_size, "LiDAR + UniPlanner pairs")
    grid = dict(min_x=dataset.min_x, max_x=dataset.max_x, min_y=dataset.min_y, max_y=dataset.max_y,
                pixels_per_meter=dataset.pixels_per_meter)
    loader = TemporalBatchLoader(dataset, batch_size, rank=rank, world=world, drop_last=False, num_workers=num_workers, ordered=True,
                                 plan_safety=plan_safety, cameras=brake, seg_model=seg_model, driving_score=driving_score)
    accs = [(Scores(), ForecastScores(), DetectedForecastScores(), PlanSafetyScores(), DetBoxScores(), BrakeScores(uni.num_cmds),
             PaintingCount(), DrivingScores(dt=step_seconds)) for _, uni in pairs]
    with math_mode(precision):
        for batch, staged in loader.staged_batches():
            actors = staged["actors"].to(dev, non_blocking=True)
            if "paint" in staged:
                for acc in accs:
                    acc[6].frames += len(staged["paint"]["pairs"])
            brake_in = None
            if brake:
                cams = staged["cameras"]
                pred_bra = brake_probs(bra, cams["rgbs"].to(dev, non_blocking=True), cams["tel"].to(dev, non_blocking=True))
                brake_in = (pred_bra, expert_track_rows(batch[10], batch[6], batch[12], batch[13], num_cmds), ctl)
            for im, acc in zip(models, accs):
                score_batch(im, batch, staged, actors, grid, acc, forecast, forecast_detected, plan_safety, det_boxes, brake_in,
                            step_seconds if driving_score else None)
    accs = gather_merged(accs)
    if accs is None:
        return None
    return [summarize(acc, precision, forecast, forecast_detected, plan_safety, dataset.num_plan, det_boxes, brake,
                      seg_model is not None, driving_score) for acc in accs]


def summarize(acc, precision, forecast, forecast_detected, plan_safety, num_plan, det_boxes=False, brake=False, painting=False,
              driving_score=False):
    """the evaluate() result of one checkpoint's accumulators ``acc`` (score_batch's tuple, then its PaintingCount and its
    DrivingScores; its DetBoxScores is read only with ``det_boxes``, its BrakeScores only with ``brake``, its PaintingCount only
    with ``painting``, its DrivingScores only with ``driving_score``)."""
    scores, forecasts, detected, safety = acc[:4]
    result = scores.summary()
    result["precision"] = precision
    if forecast:
        result["forecast"] = forecasts.summary()
    if forecast_detected:
        result["forecast_detected"] = detected.summary()
    if plan_safety:
        result["plan_safety"] = safety.summary(num_plan)
    if det_boxes:
        result["det_boxes"] = acc[4].summary()
    if brake:
        result["brake"] = acc[5].summary()
    if painting:
        result["painting"] = acc[6].summary()
    if driving_score:
        result["driving_score"] = acc[7].summary()
    return result


def score_batch(im, batch, staged, actors, grid, acc, forecast, forecast_detected, plan_safety, det_boxes=False, brake=None,
                driving_dt=None):
    """one checkpoint's InferModel ``im`` on one loader batch (its 14-tuple, staged tables and the actor table on the device),
    scored into ``acc`` = (Scores, ForecastScores, DetectedForecastScores, PlanSafetyScores, DetBoxScores, BrakeScores,
    PaintingCount, DrivingScores); the DetBoxScores is used only with ``det_boxes``, the BrakeScores only with ``brake`` = (the
    batch's brake probabilities, its expert_track_rows, the capi.ControlConfig), the DrivingScores only with a step period
    ``driving_dt``."""
    scores, forecasts, detected, safety = acc[:4]
    dev = actors.device
    lidars, num_points, bev, ego_locs, cmds, nxps = batch[0], batch[1], batch[5], batch[6], batch[7], batch[8]
    out = im.forward_batch(lidars, num_points, nxps, cmds)
    res = ops.eval_batch(out["pred_bev"].permute(0, 2, 3, 1), bev, out["packed"], actors, staged["offsets"],
                         out["ego_plan_locs"].float().contiguous(), ego_locs, grid)
    host_cmds = staged["labels"]["cmd"].numpy()
    scores.add(ops.eval_views(res.cpu(), len(num_points), out["packed"].shape[2]), host_cmds)
    if forecast:
        fc = im.uniplanner.forecast_recorded(out["features"].permute(0, 3, 1, 2), ego_locs, batch[10], batch[11], batch[12])
        k = fc["cast"].shape[0]
        forecasts.add(ops.forecast_views(score_forecasts(fc, cmds).cpu(), k + len(num_points)), k, host_cmds)
    if forecast_detected:
        h, w = out["features"].shape[1:3]                   # forward_batch's features are NHWC at half the map size
        rows = detected_rows(out["packed"].cpu().numpy(), im.pixels_per_meter, im.uniplanner.crop_centre(2 * h, 2 * w))
        res = score_detected(out, rows, actors, staged["offsets"], batch[10], ego_locs, batch[13], grid)
        detected.add(ops.det_match_views(res.cpu(), len(num_points), len(rows["col"]), batch[10].shape[2] - 1), rows["score"])
    if plan_safety:
        res = score_plan_safety(out["ego_plan_locs"], ego_locs, staged["plan_safety"], bev, grid)
        safety.add(res.cpu().numpy(), host_cmds)
    if det_boxes:
        res = ops.det_box_eval(out["packed"], actors, staged["offsets"], grid)
        acc[4].add(ops.det_box_views(res.cpu(), len(num_points), out["packed"].shape[2]))
    if brake is not None:
        pred_bra, expert, ctl = brake
        res = score_brake(out, pred_bra, expert, host_cmds.astype(np.int32), ctl)
        acc[5].add(res.cpu().numpy(), host_cmds, staged["labels"]["bra"].numpy())
    if driving_dt is not None:
        res = score_driving(out["ego_plan_locs"], ego_locs, staged["driving_score"], bev, grid, driving_dt)
        acc[7].add(res.cpu(), host_cmds)


def add_driving_score_args(ap):
    ap.add_argument("--driving-score", action="store_true",
                    help="also score the ego plan and the expert with a PDM-style driving score: at-fault collisions, drivable "
                         "area, time to collision, progress and comfort")
    ap.add_argument("--step-seconds", type=float, default=ops.DRIVING_SCORE_STEP_S,
                    help="with --driving-score: seconds between recorded frames (default %(default)s)")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config-path", default="config_v2.yaml")
    ap.add_argument("--data-dir", required=True, help="the held-out recording (replaces the YAML's data_dir)")
    add_checkpoint_args(ap, ("lidar", "uniplanner"), dict(lidar="a LiDARModel state_dict (train_full's lidar_{epoch}.th)",
                                                          uniplanner="a UniPlanner state_dict (train_full's uniplanner_{epoch}.th)"))
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--precision", default="f16", choices=["f16", "fp32"])
    ap.add_argument("--num-workers", type=int, default=16, help="host threads of the loader (record reads, PNG chunk walks)")
    ap.add_argument("--json", default=None, help="also write the result here")
    ap.add_argument("--forecast", action="store_true", help="also score the UniPlanner's forecasts of the recorded vehicles")
    ap.add_argument("--forecast-detected", action="store_true",
                    help="also score the forecasts the agent makes for the vehicles it detects, matched to the recorded tracks")
    ap.add_argument("--plan-safety", action="store_true",
                    help="also score the ego plan and the expert for collisions with the recorded traffic and for leaving the road")
    ap.add_argument("--det-boxes", action="store_true",
                    help="also score the detections as rotated boxes: IoU AP and the position, size and heading errors of the 2 m matches")
    ap.add_argument("--brake", action="store_true",
                    help="also score the agent's brake decision (brake model, plan stop, collision brake) against the recorded brake flag")
    ap.add_argument("--bra-weights", default=None, help="with --brake: the RGBBrakePredictionModel state_dict (bra_v2_9.th)")
    ap.add_argument("--agent-config", default=None,
                    help="with --brake: the agent's YAML (team_code_v2/config.yaml), for its CONTROLLER keys, cmd_thresh and "
                         "pixels_per_meter (default: --config-path)")
    ap.add_argument("--seg-weights", default=None,
                    help="paint every stacked sweep online with this RGBSegmentationModel state_dict (seg_1.th) instead of "
                         "reading the recording's lidar_sem")
    add_driving_score_args(ap)
    args = ap.parse_args(argv)
    if args.brake and args.bra_weights is None:
        ap.error("--brake needs --bra-weights")
    return args


def format_result(r):
    fmt = lambda v: "n/a" if v is None else f"{v:.4f}"
    lines = [f"{r['samples']} samples, precision {r['precision']}",
             "BEV IoU per channel: " + " ".join(fmt(v) for v in r["bev_iou"])]
    for name, d in r["det"].items():
        lines.append(f"{name} AP ({d['n_gt']} GT, {d['n_det']} detections): " + " ".join(f"{k}={fmt(v)}" for k, v in d["ap"].items()))
    p = r["plan"]
    lines.append(f"plan ADE {fmt(p['ade'])} m, FDE {fmt(p['fde'])} m")
    lines += [f"  cmd {c}: {d['samples']} samples, ADE {fmt(d['ade'])} m, FDE {fmt(d['fde'])} m" for c, d in p["per_cmd"].items()]
    if "forecast" in r:
        lines += format_forecast(r["forecast"])
    if "forecast_detected" in r:
        d = r["forecast_detected"]
        lines.append(f"forecast, detected vehicles ({d['rows']} rows, {d['matched']} matched of {d['gt']} tracked, "
                     f"{d['matched_untracked']} untracked, within {d['match_m']:g} m): recall {fmt(d['recall'])}, "
                     f"minADE {fmt(d['min_ade'])} m, minFDE {fmt(d['min_fde'])} m, top-1 ADE {fmt(d['top_ade'])} m, "
                     f"FDE {fmt(d['top_fde'])} m, miss rate {fmt(d['miss_rate'])}, AP {fmt(d['ap'])}")
    if "plan_safety" in r:
        lines += format_plan_safety(r["plan_safety"])
    if "det_boxes" in r:
        lines += format_det_boxes(r["det_boxes"])
    if "brake" in r:
        lines += format_brake(r["brake"])
    if "painting" in r:
        lines.append(f"painted online: {r['painting']['frames']} frames, {r['painting']['images']} images segmented")
    if "driving_score" in r:
        lines += format_driving_score(r["driving_score"])
    return "\n".join(lines)


def headline(r):
    """the (column, value) pairs of a result in a sweep's table."""
    cols = [(f"IoU{c}", v) for c, v in enumerate(r["bev_iou"])]
    cols += [("ped mAP", r["det"]["pedestrian"]["ap"]["mean"]), ("veh mAP", r["det"]["vehicle"]["ap"]["mean"]),
             ("ADE", r["plan"]["ade"]), ("FDE", r["plan"]["fde"])]
    if "forecast" in r:
        cols += [("fc minADE", r["forecast"]["other"]["min_ade"]), ("fc minFDE", r["forecast"]["other"]["min_fde"])]
    if "forecast_detected" in r:
        cols.append(("det fc AP", r["forecast_detected"]["ap"]))
    if "plan_safety" in r:
        cols += [("collision", r["plan_safety"]["plan"]["collision_rate"]), ("off-road", r["plan_safety"]["plan"]["off_road_rate"])]
    if "det_boxes" in r:
        veh = r["det_boxes"]["vehicle"]
        cols += [("veh AP@IoU.5", veh["ap_iou"]["0.5"]), ("veh heading", veh["heading_rad"])]
    if "brake" in r:
        agent = r["brake"]["verdicts"]["agent"]
        cols += [("false brake", agent["false_brake_rate"]), ("missed brake", agent["missed_brake_rate"])]
    if "driving_score" in r:
        cols.append(("PDMS", r["driving_score"]["plan"]["pdms"]))
    return cols


def report(checkpoints, results, world):
    """(printout, --json document) of an evaluation: one checkpoint's as format_result and its result dict; a sweep's as one
    table row per checkpoint and sweep_json."""
    if len(results) == 1:
        return format_result(results[0]), results[0]
    r0 = results[0]
    text = (f"{r0['samples']} samples, precision {r0['precision']}, {len(results)} checkpoints, {world} rank(s)\n" +
            sweep_table(checkpoints, [headline(r) for r in results]))
    return text, sweep_json(checkpoints, results, r0["samples"], world)


def main(argv=None):
    import torch.distributed as dist
    import yaml
    from .train_full import make_models
    args = parse_args(argv)
    checkpoints = select_checkpoints(args, ("lidar", "uniplanner"))
    with open(args.config_path) as f:
        cfg = yaml.safe_load(f)
    own_group = init_ranks()
    dev = eval_device()
    torch.cuda.set_device(dev)
    pairs = []
    for _, paths in checkpoints:
        # inference never runs the nested BEVPlanner: a freshly initialised one fills its place, and no bev_model_dir is read
        lid, _, uni = make_models(cfg)
        lid.load_state_dict(torch.load(paths["lidar"], map_location="cpu"))
        uni.load_state_dict(torch.load(paths["uniplanner"], map_location="cpu"))
        pairs.append((lid, uni))
    bra = agent_cfg = None
    if args.brake:
        from .heads import RGBBrakePredictionModel
        bra = RGBBrakePredictionModel(cfg["seg_channels"])
        bra.load_state_dict(torch.load(args.bra_weights, map_location="cpu"))
        if args.agent_config is not None:
            with open(args.agent_config) as f:
                agent_cfg = yaml.safe_load(f)
    seg = None
    if args.seg_weights is not None:
        from .rgb import RGBSegmentationModel
        seg = RGBSegmentationModel(cfg["seg_channels"])
        seg.load_state_dict(torch.load(args.seg_weights, map_location="cpu"))
    ds = TemporalLiDARPaintedDataset(args.config_path, device=dev, overrides=dict(data_dir=args.data_dir))
    results = evaluate_checkpoints(pairs, ds, args.batch_size, args.precision, args.num_workers, args.forecast,
                                   args.forecast_detected, args.plan_safety, args.det_boxes, args.brake, bra, agent_cfg, seg,
                                   args.driving_score, args.step_seconds)
    out = None
    if results is not None:
        text, out = report(checkpoints, results, rank_and_world()[1])
        if args.seg_weights is not None:
            out = dict(out, seg_weights=args.seg_weights)
        print(text)
        if args.json:
            with open(args.json, "w") as f:
                json.dump(out, f, indent=1)
    if own_group:
        dist.destroy_process_group()
    return out


if __name__ == "__main__":
    main()

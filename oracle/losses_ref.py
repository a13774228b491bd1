"""Float64 torch restatement of the reference trainer's encoder losses (src/ops.py, src/tf_smpl/projection.py, and the wiring of
src/trainer_sequence_fc.py compute_losses_batched / compute_losses_deltas / the e_shape part of compute_losses_prior), the oracle of
csrc/losses.cu and human_dynamics_b200/objective.py.  Gradients come from torch autograd; the optimal camera is detached.

tf.losses.absolute_difference / mean_squared_error use SUM_BY_NONZERO_WEIGHTS: the weights are broadcast to the loss's shape and the sum
is divided by the number of non-zero weights (0 when there are none).

`objective(config, inputs)` takes the same inputs as objective.Objective (a dict of tensors; the predictions stacked per set in
objective.prediction_sets order) and returns ({key: loss}, {(group, dt): optimal cameras (B, Tw, 3)}).  `nan_frames=True` keeps the
reference's NaN for an optimal-camera frame without a visible keypoint; the default gives such a frame the camera (0.7, 0, 0) and no
contribution, as the library does."""
import torch


def _safe_div(num, den):
    return num / den.clamp(min=1)          # a count of 0 has a sum of 0: the loss is 0


def absolute_difference(labels, predictions, weights):
    w = torch.broadcast_to(weights, labels.shape)
    return _safe_div((w * (labels - predictions).abs()).sum(), (w != 0).sum())


def mean_squared_error(labels, predictions, weights=None):
    if weights is None:
        weights = torch.ones((), dtype=labels.dtype, device=labels.device)
    w = torch.broadcast_to(weights, labels.shape)
    return _safe_div((w * (labels - predictions) ** 2).sum(), (w != 0).sum())


def align_by_pelvis(joints):
    pelvis = (joints[:, 3, :] + joints[:, 2, :]) / 2.
    return joints - pelvis[:, None, :]


def batch_orth_proj_idrot(X, camera):
    camera = camera.reshape(-1, 1, 3)
    return camera[:, :, 0:1] * (X[:, :, :2] + camera[:, :, 1:])


def procrustes2d_vis(X, X_target, nan_frames=False):
    """projection.py:48-104 for X (N,K,>=2), X_target (N,K,3) -> (N,3)."""
    vis = (X_target[:, :, 2] > 0).to(X.dtype)
    vv = vis[:, :, None]
    x, y = X[:, :, :2], X_target[:, :, :2]
    num = vis.sum(1, keepdim=True)[:, :, None]
    empty = (num == 0).reshape(-1)
    if not nan_frames:
        num = torch.where(num == 0, torch.ones_like(num), num)
    mu1 = (vv * x).sum(1, keepdim=True) / num
    mu2 = (vv * y).sum(1, keepdim=True) / num
    xmu = vv * (x - mu1)
    ym = vv * (y - mu2)
    A = xmu.transpose(1, 2) @ xmu + 1e-6 * torch.eye(2, dtype=X.dtype, device=X.device)
    Bm = xmu.transpose(1, 2) @ ym
    scale = torch.diagonal(torch.linalg.inv(A) @ Bm, dim1=1, dim2=2).sum(-1, keepdim=True) / 2.
    scale = scale.clamp(0.7, 10)
    trans = mu2[:, 0] / scale - mu1[:, 0]
    cam = torch.cat([scale, trans], 1)
    if not nan_frames:
        cam = torch.where(empty[:, None], torch.tensor([0.7, 0., 0.], dtype=X.dtype, device=X.device), cam)
    return cam, empty


def compute_loss_e_kp(kp_gt, kp_pred):
    kp_gt = kp_gt.reshape(-1, 3)
    kp_pred = kp_pred.reshape(-1, 2)
    return absolute_difference(kp_gt[:, :2], kp_pred, kp_gt[:, 2:3])


def compute_loss_e_kp_optcam(kp_gt, kp_pred, nan_frames=False):
    """kp_gt (B,T,K,3), kp_pred (B,T,K,2) -> (loss, best_cam (B,T,3))."""
    B, T = kp_gt.shape[:2]
    g = kp_gt.reshape(B * T, -1, 3)
    p = kp_pred.reshape(B * T, -1, 2)
    cam, empty = procrustes2d_vis(p, g, nan_frames)
    cam = cam.detach()
    proj = batch_orth_proj_idrot(p, cam)
    if not nan_frames:        # no contribution from a frame without a visible point (its weights stay in the count)
        keep = (~empty).to(p.dtype)[:, None, None]
        proj = keep * proj + (1 - keep) * g[:, :, :2].detach()
    return compute_loss_e_kp(g, proj), cam.reshape(B, T, 3)


def compute_loss_mse(params_gt, params_pred, has_gt3d):
    return 0.5 * mean_squared_error(params_gt, params_pred, has_gt3d.reshape(-1, *([1] * (params_gt.dim() - 1))))


def compute_loss_e_3d(poses_gt, poses_pred, shapes_gt, shapes_pred, joints_gt, joints_pred, batch_size, has_smpl, has_joints):
    poses_gt, poses_pred = poses_gt.reshape(batch_size, -1), poses_pred.reshape(batch_size, -1)
    shapes_gt, shapes_pred = shapes_gt.reshape(batch_size, -1), shapes_pred.reshape(batch_size, -1)
    joints_gt = align_by_pelvis(joints_gt.reshape(-1, joints_gt.shape[2], 3))
    joints_pred = align_by_pelvis(joints_pred.reshape(-1, joints_pred.shape[2], 3))
    return (compute_loss_mse(poses_gt, poses_pred, has_smpl), compute_loss_mse(shapes_gt, shapes_pred, has_smpl),
            compute_loss_mse(joints_gt, joints_pred, has_joints))


def compute_loss_e_smooth(prev, curr):
    return 0.5 * mean_squared_error(prev, curr)


def prediction_sets(config):
    """The order build_model appends the sets to pred_poses_all (trainer_sequence_fc.py:586-633): the hallucinated sets (omegas_pred_hal:
    0, then delta_t_values with do_hallucinate_preds), the prediction, the delta heads (omegas_delta)."""
    dts = [int(d) for d in config.delta_t_values]
    hal = ([('hal', 0)] + ([('hal', d) for d in dts] if config.do_hallucinate_preds else [])) if config.do_hallucinate else []
    return hal + [('pred', 0)] + ([('dt', d) for d in dts] if config.predict_delta else [])


def loss_keys(config):
    """self.losses' keys (trainer_sequence_fc.py:235-274) without the static branch."""
    keys = ['d_pose', 'e_const', 'e_joints', 'e_kp', 'e_pose', 'e_shape', 'e_smpl']
    fut_past = ['e_joints%s_future', 'e_kp%s_future', 'e_smpl%s_future', 'e_joints%s_past', 'e_kp%s_past', 'e_smpl%s_past']
    if config.predict_delta:
        keys += [k % '_dt' for k in fut_past]
    if config.do_hallucinate:
        keys += ['e_hallucinate', 'e_joints_hal', 'e_kp_hal', 'e_smpl_hal']
        if config.do_hallucinate_preds:
            keys += [k % '_hal' for k in fut_past]
    return keys


def objective(config, inputs, nan_frames=False):
    sets = prediction_sets(config)
    omega, joints, rots = inputs['omega'], inputs['joints'], inputs['rots']
    B, T, K = inputs['labels'].shape[:3]
    kps_gt = inputs['labels']
    gt_rots = inputs['gt_rots'].reshape(B, T, 24, 3, 3)
    gt_shapes = inputs['gt_shape'][:, None, :].expand(B, T, 10)
    gt3ds = inputs['gt3ds']
    hj, hs = inputs['w_joints'], inputs['w_smpl']
    losses = {k: torch.zeros((), dtype=omega.dtype, device=omega.device) for k in loss_keys(config) if k not in ('d_pose', 'e_pose')}
    cams = {}

    def pred(s):
        return {'cams': omega[s, :, :, :3], 'poses': rots[s].reshape(B, T, 24, 3, 3), 'shapes': omega[s, :, :, 75:],
                'joints': joints[s]}

    def deltas(group, suffixes):
        for s, (g, dt) in enumerate(sets):
            if g != group:
                continue
            p = pred(s)
            if dt == 0:
                sg, eg, sp, ep, L = None, None, None, None, T
            elif dt < 0:
                sg, eg, sp, ep, L = None, dt, abs(dt), None, T - abs(dt)
            else:
                sg, eg, sp, ep, L = dt, None, None, -dt, T - dt
            if dt != 0:
                kp, cam = compute_loss_e_kp_optcam(kps_gt[:, sg:eg], p['joints'][:, sp:ep, :, :2], nan_frames)
                cams[(g, dt)] = cam
            else:
                kp = compute_loss_e_kp(kps_gt[:, sg:eg], batch_orth_proj_idrot(p['joints'].reshape(B * T, K, 3),
                                                                                p['cams'].reshape(B * T, 3)))
            if config.use_3d_label:
                lp, ls, lj = compute_loss_e_3d(gt_rots[:, sg:eg], p['poses'][:, sp:ep], gt_shapes[:, sg:eg], p['shapes'][:, sp:ep],
                                               gt3ds[:, sg:eg], p['joints'][:, sp:ep, :14], B * L, hs.repeat_interleave(L),
                                               hj.repeat_interleave(L))
            else:
                lp = ls = lj = 0.
            suf = suffixes[0] if dt == 0 else (suffixes[1] if dt > 0 else suffixes[2])
            losses['e_kp' + suf] = losses['e_kp' + suf] + kp
            if config.use_3d_label:
                losses['e_joints' + suf] = losses['e_joints' + suf] + lj
                losses['e_smpl' + suf] = losses['e_smpl' + suf] + lp + ls

    if config.do_hallucinate:
        deltas('hal', ('_hal', '_hal_future', '_hal_past'))
    # compute_losses_batched
    s0 = sets.index(('pred', 0))
    p = pred(s0)
    losses['e_kp'] = compute_loss_e_kp(kps_gt, batch_orth_proj_idrot(p['joints'].reshape(B * T, K, 3), p['cams'].reshape(B * T, 3)))
    if config.use_3d_label:
        lp, ls, lj = compute_loss_e_3d(gt_rots, p['poses'], gt_shapes, p['shapes'], gt3ds, p['joints'][:, :, :14], B * T,
                                       hs.repeat_interleave(T), hj.repeat_interleave(T))
        losses['e_joints'] = lj
        losses['e_smpl'] = lp + ls
    losses['e_const'] = compute_loss_e_smooth(p['shapes'][:, :-1], p['shapes'][:, 1:]) if T > 1 else losses['e_const']
    if config.do_hallucinate:
        losses['e_hallucinate'] = mean_squared_error(inputs['strips'], inputs['pred_strips'])
    if config.predict_delta:
        deltas('dt', ('_dt', '_dt_future', '_dt_past'))
    losses['e_shape'] = (omega[:, :, :, 75:] ** 2).mean()
    return losses, cams

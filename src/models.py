"""Network entry points of the HMMR hot path -- drop-in for the reference's src/models.py.

The reference functions build TF1 graph nodes and find weights through variable scopes; these run
eagerly on float32 CUDA tensors and find weights in the active engine
(human_dynamics_b200.runtime.default_engine(), set by Tester / FeatureExtractor / HMMREngine users).
Names, argument order and return structure follow models.py (line numbers cited per function).
"""
import torch

from human_dynamics_b200 import runtime as _rt
from human_dynamics_b200.nets import run_ief_head as _run_ief_head


def get_image_encoder(model_type='resnet'):
    """models.py:12-23."""
    models = {'resnet': encoder_resnet}
    if model_type in models.keys():
        return models[model_type]
    raise ValueError('Unknown image encoder: %s' % model_type)


def get_hallucinator_model(model_type='fc2_res'):
    """models.py:26-34."""
    models = {'fc2_res': fc2_res}
    if model_type in models.keys():
        return models[model_type]
    raise ValueError('Unknown predict hal model: %s' % model_type)


def get_temporal_encoder(model_type='AZ_FC2GN'):
    """models.py:37-45."""
    models = {'AZ_FC2GN': az_fc2_groupnorm}
    if model_type in models.keys():
        return models[model_type]
    raise ValueError('Unknown temporal encoder: %s' % model_type)


def encoder_resnet(x, is_training=True, weight_decay=0.001, reuse=False):
    """Resnet v2-50 (models.py:50-77).  x: N x H x W x 3 (NHWC, [-1,1]) -> (N x 2048, 'resnet_v2_50').

    is_training=True normalises every batch norm with the moments of these N frames (the trainer's call, trainer_sequence_fc.py:562-575)
    and leaves the engine's moving averages alone, as a TF graph does without its update ops.  Forward only: no gradient flows into the
    trunk (the reference's default freeze_phi=True)."""
    eng = _rt.default_engine()
    if is_training:
        return eng.encode_images_train(x), 'resnet_v2_50'
    return eng.encode_images(x), 'resnet_v2_50'


def az_fc2_groupnorm(is_training, net, num_conv_layers):
    """f_movie: num_conv_layers x az_fc_block2 with GroupNorm (models.py:121-141).  net: B x T x 2048."""
    eng = _rt.default_engine()
    if eng.fmovie is None or len(eng.fmovie.blocks) != num_conv_layers:
        raise ValueError('active engine holds %s temporal blocks, asked for %d'
                         % (None if eng.fmovie is None else len(eng.fmovie.blocks), num_conv_layers))
    return eng.temporal_encode(net)


def fc2_res(phi, name='fc2_res'):
    """Hallucinator (models.py:270-296).  phi: B x T x 2048."""
    return _rt.default_engine().hallucinate(phi)


def _head(scope):
    eng = _rt.default_engine()
    base = 'single_view_ief'
    if scope == base:
        return eng.ief.main
    for dt, head in eng.ief.deltas.items():
        if scope == base + ('_future%d' % dt if dt > 0 else '_past%d' % abs(dt)):
            return head
    raise KeyError('no IEF weights under scope %r' % scope)


def encoder_fc3_dropout(x, num_output=85, is_training=True, reuse=False, name='3D_module', scope='single_view_ief'):
    """3 FC layers (models.py:80-116); x: N x (2048 + num_output).  Returns (delta N x num_output, None)."""
    if is_training:
        raise NotImplementedError('encoder_fc3_dropout: inference-only path (dropout is the identity)')
    head = _head(scope)
    if head.d != num_output:
        raise ValueError('scope %r regresses %d values, asked for %d' % (scope, head.d, num_output))
    phi, theta = x[:, :head.feat].contiguous(), x[:, head.feat:].contiguous()
    out = _run_ief_head(head, phi, theta, num_stage=1, impl=_rt.default_engine().impl)
    return out - theta, None


def hmr_ief(phi, omega_start, scope, num_output=85, num_stage=3, is_training=True):
    """HMR-style IEF (models.py:380-415): phi N x 2048, omega_start N x num_output -> N x num_output."""
    if is_training:
        raise NotImplementedError('hmr_ief: inference-only path')
    head = _head(scope)
    if head.d != num_output:
        raise ValueError('scope %r regresses %d values, asked for %d' % (scope, head.d, num_output))
    return _run_ief_head(head, phi.contiguous(), omega_start, num_stage=num_stage, impl=_rt.default_engine().impl)


def call_hmr_ief(phi, omega_start, scope, num_output=85, num_stage=3, is_training=True, predict_delta_keys=(),
                 use_delta_from_pred=False, use_optcam=True):
    """models.py:299-377.  Returns (theta N x num_output, {delta_t: N x 85})."""
    theta_here = hmr_ief(phi, omega_start, scope, num_output, num_stage, is_training)
    num_output_delta = 72 if use_optcam else 3 + 72
    deltas_predictions = {}
    for delta_t in predict_delta_keys:
        if delta_t == 0:
            continue
        scope_delta = scope + ('_future{}'.format(delta_t) if delta_t > 0 else '_past{}'.format(abs(delta_t)))
        omega_start_delta = theta_here if use_delta_from_pred else omega_start
        beta = omega_start_delta[:, -10:]
        if use_optcam:
            omega_start_delta = omega_start_delta[:, 3:3 + num_output_delta]
        else:
            omega_start_delta = omega_start_delta[:, :num_output_delta]
        delta_pred = hmr_ief(phi, omega_start_delta, scope_delta, num_output_delta, num_stage, is_training)
        n = delta_pred.shape[0]
        if use_optcam:      # plumbing: assemble [1, 0, 0, pose72, beta]  (models.py:367-371)
            out = torch.empty((n, 85), dtype=torch.float32, device=delta_pred.device)
            out[:, 0] = 1.0
            out[:, 1:3] = 0.0
            out[:, 3:75] = delta_pred
            out[:, 75:] = beta
            delta_pred = out
        else:
            delta_pred = torch.cat([delta_pred[:, :75], beta], 1)
        deltas_predictions[delta_t] = delta_pred
    return theta_here, deltas_predictions


def batch_pred_omega(input_features, batch_size, is_training, num_output, omega_mean, sequence_length, scope,
                     predict_delta_keys=(), use_delta_from_pred=False, use_optcam=False):
    """models.py:233-267: B x T x * features -> (B x T x num_output, {delta_t: B x T x num_output})."""
    feats = input_features.reshape(batch_size * sequence_length, -1)
    eng = _rt.default_engine()
    keys = tuple(sorted(int(k) for k in predict_delta_keys if int(k) != 0))
    fast = (scope == 'single_view_ief' and num_output == 85 and use_optcam and use_delta_from_pred and not is_training
            and all(k in eng.ief.deltas for k in keys))
    if fast:        # the Tester wiring (tester.py:196-207): cached plan, no per-call binding
        omega_pred, deltas = eng.regress(feats, omega_start=omega_mean, delta_keys=keys)
    else:
        omega_pred, deltas = call_hmr_ief(feats, omega_mean, scope, num_output, 3, is_training, predict_delta_keys,
                                          use_delta_from_pred, use_optcam)
    omega_pred = omega_pred.reshape(batch_size, sequence_length, num_output)
    return omega_pred, {k: v.reshape(batch_size, sequence_length, num_output) for k, v in deltas.items()}

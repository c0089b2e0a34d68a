"""The objective training/v2/training.py minimises, for a v2 checkpoint on one batch, on the device.

    batch = datareader.build_batch(pool, pairs, params, augmentation)   # IMAGE_PAIR, MOTION, DEPTH, INTRINSICS
    losses = objective(session, batch, '3_dm2')
    losses['netDM2_loss_depth2'], losses['regularization'], losses['total']   # 0-d torch CUDA tensors

For one of training.py's evolutions this builds what its tower builds and returns the losses it adds to the total:
  * preprocessing (training.py:170-184): prepare_ground_truth_tensors(DEPTH, MOTION[:, :3], MOTION[:, 3:], INTRINSICS),
    image2_2 = resize_area(image2, 48x64), image1 for 5_refine;
  * blocks (training.py:190-436): netFlow1 always, netDM1 from 1_dm1, netFlow2 from 2_flow2 on INTRINSICS and netDM1's
    predictions, netDM2 from 3_dm2 on netFlow2's flow and netDM1's motion, netRefine at 5_refine (v2.blocks);
  * the selected losses of each evolution, SELECTED_LOSSES (training.py:227, 273, 373, 425, 456), under their prefixes;
  * 'regularization' (training.py:75, 491-495): 0.0004 * sum of tf.nn.l2_loss over the kernels of every block the
    evolution builds.  v2/blocks.py passes kernel_regularizer to every conv, transposed conv and dense layer, and
    get_regularization_losses(scope=tower) collects the losses of all of them, trained or not, because each is created
    under the tower's name scope.  The sum depends on the checkpoint only: Session.kernel_l2, float64 from the host copy;
  * 'total': the selected losses in training.py's order, then the regularisation (tf.add_n of training.py:495).

Weights.  training.py schedules flow_sig_weight, conf_sig_weight, level5_factor and depth_sig_weight with tfutils'
ease_out_quad / ease_in_quad, whose curves the reference does not include.  They are arguments here, and their defaults
are the values each schedule ends at: the full gradient weights, level5_factor = 0, and half of _depth_grad_loss_weight
for netRefine.  The fixed weights default to training.py's constants.

4_iterative and 5_refine.  training.py appends to each batch of 8 the 24 samples of earlier iterations from a FIFO queue
(training.py:278-321); netFlow1 and netDM1 see only the 8 new ones, and netFlow2's previous predictions are netDM1's for
those 8 followed by the queue's for the rest.  The queue is not built here.  `batch` is the whole tower batch (new samples
first), and `prev_predictions` holds predict_depth2, predict_normal2, predict_rotation and predict_translation of its last
rows, the earlier iterations' results; netFlow1 and netDM1 run on the rows before them.  Without it netFlow1 and netDM1
run on every row and netFlow2 starts from their results, which is what the queue holds when training starts
(training.py:301-311).

The result is a dict of 0-d torch CUDA tensors in the networks' float32, computed without a host synchronisation.
"""
import torch

from .. import images
from . import blocks, losses, networks as _nets

EVOLUTIONS = ('0_flow1', '1_dm1', '2_flow2', '3_dm2', '4_iterative', '5_refine')
SCOPES = ('netFlow1', 'netDM1', 'netFlow2', 'netDM2', 'netRefine')

_FLOW = ('loss_flow5', 'loss_flow2', 'loss_flow2_sig', 'loss_conf5', 'loss_conf2', 'loss_conf2_sig')
_DM = ('loss_depth2', 'loss_depth2_sig', 'loss_normal2', 'loss_rotation', 'loss_translation')
_REFINE = ('loss_depth0', 'loss_depth0_sig', 'loss_normal0')

# evolution -> ((loss_prefix, selected_losses), ...) in the order training.py adds them to the 'losses' collection
SELECTED_LOSSES = {
    '0_flow1': (('netFlow1_', _FLOW),),
    '1_dm1': (('netDM1_', _DM),),
    '2_flow2': (('netFlow2_', _FLOW),),
    '3_dm2': (('netDM2_', _DM),),
    '4_iterative': (('netFlow2_', _FLOW), ('netDM2_', _DM)),
    '5_refine': (('netRefine_', _REFINE),),
}

REGULARIZATION_SCALE = 0.0004   # tf.contrib.layers.l2_regularizer(0.0004), training.py:75

# training.py:66-74 and the end points of its schedules
DEFAULT_WEIGHTS = {
    'flow_weight': 0.5 * 1000, 'conf_weight': 0.5 * 100 * 0.5, 'flow_sig_weight': 0.25 * 1000, 'conf_sig_weight': 0.25 * 100,
    'level5_factor': 0, 'depth_weight': 0.5 * 300, 'depth_sig_weight': 0.25 * 1500, 'normal_weight': 0.5 * 50,
    'rotation_weight': 160, 'translation_weight': 15 * 3,
}
_PREV = ('predict_depth2', 'predict_normal2', 'predict_rotation', 'predict_translation')


def built_scopes(evolution):
    """The blocks training.py builds at `evolution` (training.py:190-436)."""
    i = EVOLUTIONS.index(evolution)
    return SCOPES[:min(i, 3) + 1] + (('netRefine',) if evolution == '5_refine' else ())


def regularization(session, evolution):
    """0.0004 * sum of l2_loss(kernel) over the built blocks, as a Python float (float64)."""
    l2 = session.kernel_l2()
    return REGULARIZATION_SCALE * sum(l2[s] for s in built_scopes(evolution))


def _weights(evolution, weights):
    unknown = sorted(set(weights) - set(DEFAULT_WEIGHTS))
    if unknown:
        raise TypeError("objective() got an unexpected weight %r (known: %s)" % (unknown[0], ", ".join(sorted(DEFAULT_WEIGHTS))))
    w = dict(DEFAULT_WEIGHTS)
    if evolution == '5_refine':
        w['depth_sig_weight'] = 0.5 * DEFAULT_WEIGHTS['depth_sig_weight']   # training.py:440
    w.update(weights)
    return w


def _flow_losses(res, gt, w, prefix):
    """training.py:195-223"""
    fc5, fc2 = res['predict_flowconf5'], res['predict_flowconf2']
    return losses.flow_loss_block(gt['flow2'], gt['flow5'], gt['flow2_sig'], fc2[:, 0:2], fc5[:, 0:2], fc2[:, 2:4], fc5[:, 2:4],
                                  w['flow_weight'], w['conf_weight'], w['flow_sig_weight'], w['conf_sig_weight'], conf_diff_scale=10,
                                  level5_factor=w['level5_factor'], loss_prefix=prefix)


def _dm_losses(res, gt, w, prefix):
    """training.py:252-269"""
    return losses.depthnormal_loss_block(gt['depth2'], gt['depth2_sig'], gt['normal2'], gt['rotation'], gt['translation'],
                                         res['predict_depth2'], res['predict_normal2'], res['predict_rotation'],
                                         res['predict_translation'], w['depth_weight'], w['depth_sig_weight'], w['normal_weight'],
                                         w['rotation_weight'], w['translation_weight'], translation_factor=1, loss_prefix=prefix)


def _cuda(x, name):
    t = x if isinstance(x, torch.Tensor) else torch.as_tensor(x)
    if not t.is_cuda:
        t = t.cuda()
    if t.dtype != torch.float32:
        raise TypeError("batch[%r] must be float32, got %s" % (name, t.dtype))
    return t.contiguous()


def objective(session, batch, evolution, prev_predictions=None, **weights):
    """training.py's selected losses, 'regularization' and 'total' for `evolution` on `batch` (a dict with IMAGE_PAIR
    [B,6,192,256], MOTION [B,6] angle-axis rotation ++ translation, DEPTH [B,1,192,256] inverse depth and INTRINSICS [B,4],
    as datareader.build_batch makes them).  `weights` override DEFAULT_WEIGHTS."""
    if evolution not in EVOLUTIONS:
        raise ValueError("evolution must be one of %s, got %r" % (", ".join(EVOLUTIONS), evolution))
    w = _weights(evolution, weights)
    session = session if session is not None else _nets.default_session()
    ip, motion, depth, K = (_cuda(batch[k], k) for k in ('IMAGE_PAIR', 'MOTION', 'DEPTH', 'INTRINSICS'))
    B = int(ip.shape[0])
    new = B
    if prev_predictions is not None:
        if evolution < '4_iterative':
            raise ValueError("prev_predictions: only 4_iterative and 5_refine take earlier iterations, not %s" % evolution)
        for k in _PREV:
            if k not in prev_predictions:
                raise ValueError("prev_predictions has no %s" % k)
        new = B - int(prev_predictions['predict_rotation'].shape[0])
        if new < 1:
            raise ValueError("prev_predictions has %d rows; the batch of %d needs at least one new sample"
                             % (B - new, B))

    # data preprocessing, training.py:170-184
    rotation, translation = motion[:, 0:3].contiguous(), motion[:, 3:6].contiguous()
    gt = losses.prepare_ground_truth_tensors(depth, rotation, translation, K)
    gt['rotation'], gt['translation'] = rotation, translation
    image2_2 = images.resize_area(ip[:, 3:6], (48, 64))

    got = {}
    flow1 = blocks.flow_block(ip[:new], scope='netFlow1', session=session)
    if evolution == '0_flow1':
        got.update(_flow_losses(flow1, gt, w, 'netFlow1_'))
    if evolution >= '1_dm1':
        fc2 = flow1['predict_flowconf2']
        dm1 = blocks.depthmotion_block(ip[:new], image2_2[:new], fc2[:, 0:2], fc2, scope='netDM1', session=session)
    if evolution == '1_dm1':
        got.update(_dm_losses(dm1, gt, w, 'netDM1_'))
    if evolution >= '2_flow2':
        prev = {k: dm1[k] if prev_predictions is None else torch.cat((dm1[k], _cuda(prev_predictions[k], k)), dim=0) for k in _PREV}
        flow2 = blocks.flow_block(ip, image2_2, K, prev, scope='netFlow2', session=session)
    if evolution in ('2_flow2', '4_iterative'):
        got.update(_flow_losses(flow2, gt, w, 'netFlow2_'))
    if evolution >= '3_dm2':
        fc2 = flow2['predict_flowconf2']
        dm2 = blocks.depthmotion_block(ip, image2_2, fc2[:, 0:2], fc2, prev['predict_rotation'], prev['predict_translation'], K,
                                       scope='netDM2', session=session)
    if evolution in ('3_dm2', '4_iterative'):
        got.update(_dm_losses(dm2, gt, w, 'netDM2_'))
    if evolution == '5_refine':
        ref = blocks.depth_refine_block(ip[:, 0:3], dm2, session=session)
        got.update(losses.depth_refine_loss_block(gt['depth0'], gt['depth0_sig'], gt['normal0'], ref['predict_depth0'],
                                                  ref['predict_normal0'], w['depth_weight'], w['depth_sig_weight'],
                                                  w['normal_weight'], loss_prefix='netRefine_'))

    out = {}
    for prefix, names in SELECTED_LOSSES[evolution]:
        for name in names:
            out[prefix + name] = got[prefix + name]
    out['regularization'] = torch.full((), regularization(session, evolution), dtype=torch.float32, device=ip.device)
    total = None
    for v in out.values():
        total = v if total is None else total + v
    out['total'] = total
    return out

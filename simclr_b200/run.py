"""Pretraining driver: the flag surface and `single_step` of the reference's
`tf2/run.py` on the H100 engine.

`python -m simclr_b200.run --train_batch_size=512 ...` (under torchrun for more
than one GPU: one process per GPU, NCCL over NVLink) trains on synthetic
tensors of the reference's input contract (`tf2/data.py:52-62`: [B,H,W,6] fp32 in
[0,1] + one-hot labels), with the reference's modes (train / eval / train_then_eval,
pretrain / finetune), checkpoint cadence and TensorBoard metrics; dataset reading (TFDS)
and SavedModel export are outside this path (SURVEY.md section 8).
"""
import json
import math
import os

import torch
import torch.distributed as dist
from absl import app
from absl import logging

from .flags_def import FLAGS
from . import engine as engine_lib
from . import model as model_lib
from . import objective as obj_lib
from ._lib import lib, stream_ptr


class Trainer:
    """Owns model + optimizer and runs `single_step` (tf2/run.py:557-622)."""

    def __init__(self, num_classes=None, num_examples=None, seed=0, engine=None):
        self.engine = engine or engine_lib.get_engine()
        self.strategy = self.engine.ctx
        self.num_classes = num_classes or FLAGS.b200_num_classes
        self.num_examples = num_examples or FLAGS.b200_num_examples
        self.model = model_lib.Model(self.num_classes, seed=seed)
        self.learning_rate = model_lib.WarmUpAndCosineDecay(FLAGS.learning_rate, self.num_examples)
        self.optimizer = model_lib.build_optimizer(self.learning_rate)
        self.metrics = {}
        self._graph = None
        self._graph_bottom = None
        self._graph_apply = None
        self._static = None
        self._bw_state = None
        self._split_off = None
        self._side = None
        self._top_work = None

    # ------------------------------------------------------------------
    GRAD_SPLIT = 2      # backward_top covers block groups 3-4 + heads: 96 % of the ResNet-50 gradient bytes

    def single_step(self, features, labels):
        """One synchronous data-parallel step on this replica's shard.

        features [B,H,W,6] fp32, labels one-hot [B,classes] fp32 (or None).
        Loss = contrastive + supervised + weight decay, divided by the number of
        replicas (tf2/run.py:587-617); gradients are summed across replicas
        (Keras `apply_gradients`, C3) and LARS is applied.  With more than one replica the gradient
        all-reduce of the late layers runs on a side stream under the backward pass of the early ones."""
        if self._overlap_ok():
            loss = self.forward_backward_top(features, labels)
            self.reduce_gradients_top_async()
            self.backward_bottom()
            self.reduce_gradients_bottom()
        else:
            loss = self.forward_backward(features, labels)
            self.reduce_gradients()
        self.optimizer.apply_gradients([(v.grad, v) for v in self.model.trainable_variables])
        return loss

    def _overlap_ok(self):
        if self.strategy.num_replicas_in_sync < 2 or FLAGS.train_mode != 'pretrain' or 'lars' not in FLAGS.optimizer:
            return False
        if os.environ.get('SIMCLR_GRAD_OVERLAP', '1') == '0':
            return False
        if self._split_off is None:
            off = self.model.grad_split_offset(self.GRAD_SPLIT)
            self._split_off = off if off else -1
        return self._split_off > 0

    def forward_backward(self, features, labels):
        """Forward, losses and the explicit backward pass: fills `.grad` of every trainable
        variable with THIS replica's contribution.  The collectives inside (SyncBN statistics,
        embedding / log-sum-exp all-gathers) are our own peer-memory kernels when
        `strategy.comm` is set, so this part is CUDA-graph capturable at any replica count."""
        loss = self.forward_backward_top(features, labels, split=0)
        self.backward_bottom(split=0)
        return loss

    def forward_backward_top(self, features, labels, split=None):
        """Forward, losses, and the backward pass down to block group `split`+1 (all of it for split 0)."""
        e, model = self.engine, self.model
        split = self.GRAD_SPLIT if split is None else split
        e.begin_step(model.vs.flat_grad)       # BN-sum pool and the flat gradient buffer zeroed once
        try:
            return self._forward_backward_top(features, labels, split)
        except BaseException:
            e.end_step()
            raise

    def backward_bottom(self, split=None):
        split = self.GRAD_SPLIT if split is None else split
        try:
            self.model.backward_bottom(self._bw_state, split)
            if 'lars' not in FLAGS.optimizer:       # every gradient is final now
                R = self.strategy.num_replicas_in_sync
                for v in self.model.trainable_variables:
                    if 'batch_normalization' not in v.name and v.grad is not None:
                        lib.axpy(float(FLAGS.weight_decay) / R, v.value, v.grad, v.numel, stream_ptr())
        finally:
            self._bw_state = None
            self.engine.end_step()

    def _forward_backward_top(self, features, labels, split):
        e, model, R = self.engine, self.model, self.strategy.num_replicas_in_sync
        st = stream_ptr()
        projection_head_outputs, supervised_head_outputs = model(features, training=True)
        B = features.shape[0]
        loss = None
        d_proj = d_sup = None
        if projection_head_outputs is not None:
            con_loss, logits_con, labels_con, ctx = obj_lib.contrastive_forward(
                projection_head_outputs, hidden_norm=FLAGS.hidden_norm, temperature=FLAGS.temperature,
                strategy=self.strategy if R > 1 else None, want_labels=False)
            loss = con_loss
            d_proj = obj_lib.contrastive_backward(ctx, 1.0 / (B * R))
            self.metrics['contrast_loss'] = con_loss
            self.metrics['logits_con'] = logits_con
        if supervised_head_outputs is not None:
            # l = concat([l, l], 0) (tf2/run.py:600-602): row r uses labels[r % B]
            sup_loss, d_sup = obj_lib.add_supervised_loss(labels, supervised_head_outputs,
                                                          grad_scale=1.0 / (supervised_head_outputs.shape[0] * R))
            loss = sup_loss if loss is None else loss + sup_loss
            self.metrics['supervised_loss'] = sup_loss
            self.metrics['supervised_logits'] = supervised_head_outputs
        weight_decay = model_lib.add_weight_decay(model, adjust_per_optimizer=True)
        self.metrics['weight_decay'] = weight_decay
        loss = loss + weight_decay
        self.metrics['total_loss'] = loss
        self._bw_state = model.backward_top(d_proj, d_sup, split)
        # d(weight_decay)/dW = wd * W (loss / R per replica): with LARS on the supervised-head kernel only (the
        # optimizer decays the rest; its gradient is final here), otherwise on every non-BatchNorm variable
        # (tf2/model.py:47-69) -- those runs do not split the backward pass
        assert split == 0 or 'lars' in FLAGS.optimizer
        if 'lars' in FLAGS.optimizer:
            for v in model.trainable_variables:
                if 'head_supervised' in v.name and 'bias' not in v.name and v.grad is not None:
                    lib.axpy(float(FLAGS.weight_decay) / R, v.value, v.grad, v.numel, st)
        return loss

    def reduce_gradients(self):
        """C3: cross-replica SUM of the gradients, one NCCL all-reduce over the flat buffer."""
        if self.strategy.num_replicas_in_sync > 1:
            self.strategy.all_reduce_sum(self.model.vs.flat_grad)

    def reduce_gradients_top_async(self):
        """All-reduce of the gradients `forward_backward_top` has finished (block groups 3-4 + heads: the tail of
        the flat buffer) on a side stream: it runs under `backward_bottom`."""
        if self._side is None:
            self._side = torch.cuda.Stream()
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        with torch.cuda.stream(self._side):
            self._side.wait_event(ev)
            self._top_work = dist.all_reduce(self.model.vs.flat_grad[self._split_off:], op=dist.ReduceOp.SUM,
                                             group=self.strategy.group, async_op=True)

    def reduce_gradients_bottom(self):
        dist.all_reduce(self.model.vs.flat_grad[:self._split_off], op=dist.ReduceOp.SUM, group=self.strategy.group)
        self._top_work.wait()                   # the current stream waits for the side-stream all-reduce
        torch.cuda.current_stream().wait_stream(self._side)
        self._top_work = None

    # ------------------------------------------------------------------
    def capture(self, features, labels, warmup=2, restore=False):
        """Captures `single_step` in a CUDA graph (the reference runs its steps inside
        one `tf.while_loop`, tf2/run.py:626-638).  `features`/`labels` become the
        static input buffers: copy new data into them before `replay()`.

        The `warmup` eager steps run on a side stream first (lazy initialisation, allocator
        warm-up) and are REAL steps: they update weights, momentum, moving statistics and
        advance `optimizer.iterations`.  `restore=True` snapshots that state before the
        warm-up and puts it back after the capture, so the first `replay()` is step
        `optimizer.iterations` of the schedule on the pre-capture weights.  The capture
        itself executes nothing and does not advance the schedule."""
        self._static = (features, labels)
        opt, vs = self.optimizer, self.model.vs
        opt.ensure_built(self.model.trainable_variables)      # H2D table copies must not land in the capture
        snap = None
        if restore:
            snap = (vs.flat_value.clone(), vs.flat_moving.clone(), opt._flat_v.clone(), opt.iterations)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self.single_step(features, labels)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.optimizer.stage_learning_rate()
        R = self.strategy.num_replicas_in_sync
        if R == 1:
            self._graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph):
                self._graph_loss = self.single_step(features, labels)
            self._graph_apply = None
        else:
            # More than one replica: the in-step collectives are peer-memory kernels (capturable); the
            # gradient all-reduce is NCCL and stays between two graphs.
            if self.strategy.comm is None:
                raise RuntimeError('CUDA-graph capture with %d replicas needs the peer-memory collectives '
                                   '(strategy.comm); run eagerly instead' % R)
            self._graph = torch.cuda.CUDAGraph()
            self._graph_bottom = None
            if self._overlap_ok():
                # three graphs: [forward + backward of groups 3-4 and heads] | all-reduce of their gradients on a side
                # stream, under [backward of groups 1-2 and the stem] | all-reduce of the rest | [LARS]
                with torch.cuda.graph(self._graph):
                    self._graph_loss = self.forward_backward_top(features, labels)
                self._graph_bottom = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self._graph_bottom, pool=self._graph.pool()):
                    self.backward_bottom()
            else:
                with torch.cuda.graph(self._graph):
                    self._graph_loss = self.forward_backward(features, labels)
            self._graph_apply = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph_apply, pool=self._graph.pool()):
                self.optimizer.apply_gradients([(v.grad, v) for v in self.model.trainable_variables])
        if snap is not None:
            vs.flat_value.copy_(snap[0]); vs.flat_moving.copy_(snap[1]); opt._flat_v.copy_(snap[2])
            opt.iterations = snap[3]
        return self._graph

    def replay(self):
        self.optimizer.prepare_replay()
        self._graph.replay()
        if self._graph_apply is not None:
            if self._graph_bottom is not None:
                self.reduce_gradients_top_async()
                self._graph_bottom.replay()
                self.reduce_gradients_bottom()
            else:
                self.reduce_gradients()
            self._graph_apply.replay()
        return self._graph_loss


def init_distributed():
    """One process per GPU under torchrun; no-op for a single process."""
    if 'RANK' in os.environ and int(os.environ.get('WORLD_SIZE', '1')) > 1 and not dist.is_initialized():
        local_rank = int(os.environ.get('LOCAL_RANK', '0'))
        torch.cuda.set_device(local_rank)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
    return dist.get_rank() if dist.is_initialized() else 0


def synthetic_batch(batch, image_size, num_classes, device, seed):
    """Synthetic inputs of the reference's input contract (SURVEY.md 8d)."""
    g = torch.Generator(device=device).manual_seed(seed)
    features = torch.rand(batch, image_size, image_size, 6, device=device, generator=g)
    idx = torch.randint(0, num_classes, (batch,), device=device, generator=g)
    labels = torch.nn.functional.one_hot(idx, num_classes).float()
    return features, labels


def synthetic_eval_batch(batch, image_size, num_classes, device, seed):
    """One view per sample, the contract of the eval / finetune pipeline (tf2/data.py:52-62 with
    is_pretrain False): [B,H,W,3] fp32 in [0,1] + one-hot labels."""
    g = torch.Generator(device=device).manual_seed(seed)
    features = torch.rand(batch, image_size, image_size, 3, device=device, generator=g)
    idx = torch.randint(0, num_classes, (batch,), device=device, generator=g)
    return features, torch.nn.functional.one_hot(idx, num_classes).float()


def json_serializable(val):
    try:
        json.dumps(val)
        return True
    except TypeError:
        return False


def perform_evaluation(trainer, eval_steps, ckpt, batch_fn):
    """tf2/run.py:348-432: restores `ckpt`, runs `eval_steps` inference steps (BatchNorm on moving statistics),
    accumulates eval/regularization_loss and label top-1 / top-5 accuracy, writes the TensorBoard summaries,
    result.json, result_<step>.json and flags.json into model_dir.  `batch_fn(i)` -> (features, one-hot labels)."""
    from . import metrics as metrics_lib, checkpoint as ckpt_lib
    if FLAGS.train_mode == 'pretrain' and not FLAGS.lineareval_while_pretraining:
        logging.info('Skipping eval during pretraining without linear eval.')
        return None
    model = trainer.model
    regularization_loss = metrics_lib.Mean('eval/regularization_loss')
    label_top_1_accuracy = metrics_lib.Accuracy('eval/label_top_1_accuracy')
    label_top_5_accuracy = metrics_lib.TopKCategoricalAccuracy(5, 'eval/label_top_5_accuracy')
    all_metrics = [regularization_loss, label_top_1_accuracy, label_top_5_accuracy]
    global_step = 0
    if ckpt:
        logging.info('Restoring from %s', ckpt)
        global_step = ckpt_lib.CheckpointManager(model, None, FLAGS.model_dir).restore(ckpt)
        logging.info('Performing eval at step %d', global_step)
    for i in range(eval_steps):
        features, labels = batch_fn(i)
        _, supervised_head_outputs = model(features, training=False)
        assert supervised_head_outputs is not None
        metrics_lib.update_finetune_metrics_eval(label_top_1_accuracy, label_top_5_accuracy, supervised_head_outputs, labels)
        regularization_loss.update_state(model_lib.add_weight_decay(model, adjust_per_optimizer=True))
        logging.info('Completed eval for %d / %d steps', i + 1, eval_steps)
    result = {m.name: float(m.result()) for m in all_metrics}
    result['global_step'] = int(global_step)
    logging.info(result)
    if FLAGS.model_dir and trainer.strategy.replica_id == 0:
        writer = metrics_lib.SummaryWriter(FLAGS.model_dir)
        metrics_lib.log_and_write_metrics_to_summary(all_metrics, global_step, writer)
        writer.flush(); writer.close()
        for name in ('result.json', 'result_%d.json' % result['global_step']):
            with open(os.path.join(FLAGS.model_dir, name), 'w') as f:
                json.dump({k: float(v) for k, v in result.items()}, f)
        with open(os.path.join(FLAGS.model_dir, 'flags.json'), 'w') as f:
            json.dump({k: v for k, v in FLAGS.flag_values_dict().items() if json_serializable(v)}, f)
    return result


def main(argv):
    """tf2/run.py:464-664 on synthetic tensors: `--mode=train|eval|train_then_eval`, `--train_mode=pretrain|finetune`,
    checkpoints every `checkpoint_steps` (resume from the latest one in --model_dir, or weights from --checkpoint),
    train/* metrics + learning rate flushed to TensorBoard event files at the same cadence.  Reading a dataset
    (TFDS) and SavedModel export are not part of this path (SURVEY.md section 8: N1 / N2)."""
    from . import metrics as metrics_lib, checkpoint as ckpt_lib
    if len(argv) > 1:
        raise app.UsageError('Too many command-line arguments.')
    rank = init_distributed()
    engine_lib.set_engine(engine_lib.Engine())
    # --data_dir: a prepared TFDS directory (TFRecord shards, data.TFRecordBuilder), or an .npz of decoded images
    # (data.ArrayBuilder.from_npz); without it: synthetic tensors of the input contract
    builder = None
    if FLAGS.data_dir:
        from . import data as data_lib
        npz = FLAGS.data_dir if os.path.isfile(FLAGS.data_dir) else os.path.join(FLAGS.data_dir, FLAGS.dataset + '.npz')
        if os.path.isfile(npz):
            builder = data_lib.ArrayBuilder.from_npz(npz)
        else:
            builder = data_lib.TFRecordBuilder(FLAGS.data_dir, FLAGS.dataset)
        builder.download_and_prepare()
        trainer = Trainer(num_classes=builder.info.features['label'].num_classes,
                          num_examples=builder.info.splits[FLAGS.train_split].num_examples)
    else:
        trainer = Trainer()
    R = trainer.strategy.num_replicas_in_sync
    dev = trainer.engine.device
    num_train_examples, num_classes = trainer.num_examples, trainer.num_classes
    num_eval_examples = (builder.info.splits[FLAGS.eval_split].num_examples if builder is not None
                         else FLAGS.b200_num_eval_examples)
    train_steps = model_lib.get_train_steps(num_train_examples)
    eval_steps = FLAGS.eval_steps or int(math.ceil(num_eval_examples / FLAGS.eval_batch_size))
    epoch_steps = int(round(num_train_examples / FLAGS.train_batch_size))
    checkpoint_steps = FLAGS.checkpoint_steps or (FLAGS.checkpoint_epochs * epoch_steps)
    logging.info('# train examples: %d', num_train_examples)
    logging.info('# train_steps: %d', train_steps)
    logging.info('# eval examples: %d', num_eval_examples)
    logging.info('# eval steps: %d', eval_steps)
    assert FLAGS.eval_batch_size % R == 0 and FLAGS.train_batch_size % R == 0
    if builder is not None:
        def eval_fn(i, _it=[None]):
            if i == 0 or _it[0] is None:
                _it[0] = data_lib.build_distributed_dataset(builder, FLAGS.eval_batch_size, False, trainer.strategy, None)
            return next(_it[0])
    else:
        eval_fn = lambda i: synthetic_eval_batch(FLAGS.eval_batch_size // R, FLAGS.image_size, num_classes, dev, 99991 * (rank + 1) + i)

    if FLAGS.mode == 'eval':
        manager = ckpt_lib.CheckpointManager(trainer.model, None, FLAGS.model_dir)
        result = perform_evaluation(trainer, eval_steps, manager.latest_checkpoint, eval_fn)
        logging.info('Eval complete. Exiting...')
        if dist.is_initialized():
            dist.destroy_process_group()
        return result

    B = FLAGS.train_batch_size // R            # per-replica batch size (tf2/data.py:45)
    pretrain = FLAGS.train_mode == 'pretrain'
    writer = metrics_lib.SummaryWriter(FLAGS.model_dir) if (FLAGS.model_dir and rank == 0) else None
    weight_decay_metric = metrics_lib.Mean('train/weight_decay')
    total_loss_metric = metrics_lib.Mean('train/total_loss')
    all_metrics = [weight_decay_metric, total_loss_metric]
    if pretrain:
        contrast_loss_metric = metrics_lib.Mean('train/contrast_loss')
        contrast_acc_metric = metrics_lib.Mean('train/contrast_acc')
        contrast_entropy_metric = metrics_lib.Mean('train/contrast_entropy')
        all_metrics.extend([contrast_loss_metric, contrast_acc_metric, contrast_entropy_metric])
    if not pretrain or FLAGS.lineareval_while_pretraining:
        supervised_loss_metric = metrics_lib.Mean('train/supervised_loss')
        supervised_acc_metric = metrics_lib.Mean('train/supervised_acc')
        all_metrics.extend([supervised_loss_metric, supervised_acc_metric])
    manager = ckpt_lib.try_restore_from_checkpoint(trainer.model, trainer.optimizer) if FLAGS.model_dir else None
    steps_per_loop = max(1, checkpoint_steps)
    cur_step = trainer.optimizer.iterations
    iterator = (data_lib.build_distributed_dataset(builder, FLAGS.train_batch_size, True, trainer.strategy, None)
                if builder is not None else None)
    while cur_step < train_steps:
        for _ in range(min(steps_per_loop, train_steps - cur_step)):
            seed = 1234 + rank + 7919 * cur_step
            if iterator is not None:
                features, labels = next(iterator)
            elif pretrain:
                features, labels = synthetic_batch(B, FLAGS.image_size, num_classes, dev, seed)
            else:
                features, labels = synthetic_eval_batch(B, FLAGS.image_size, num_classes, dev, seed)
            loss = trainer.single_step(features, labels)
            m = trainer.metrics
            weight_decay_metric.update_state(m['weight_decay'])
            total_loss_metric.update_state(m['total_loss'])
            if pretrain:
                metrics_lib.update_pretrain_metrics_train(contrast_loss_metric, contrast_acc_metric, contrast_entropy_metric,
                                                          m['contrast_loss'], m['logits_con'], None,
                                                          trainer.strategy.replica_id)
            if 'supervised_loss' in m:
                metrics_lib.update_finetune_metrics_train(supervised_loss_metric, supervised_acc_metric,
                                                          m['supervised_loss'], labels, m['supervised_logits'])
            cur_step = trainer.optimizer.iterations
        if manager is not None and rank == 0:
            manager.save(cur_step)
        logging.info('Completed: %d / %d steps', cur_step, train_steps)
        if rank == 0:
            metrics_lib.log_and_write_metrics_to_summary(all_metrics, cur_step, writer)
            if writer is not None:
                writer.scalar('learning_rate', trainer.learning_rate(cur_step), cur_step)
                writer.flush()
        for metric in all_metrics:
            metric.reset_states()
    logging.info('Training complete...')
    result = None
    if FLAGS.mode == 'train_then_eval':
        result = perform_evaluation(trainer, eval_steps, manager.latest_checkpoint if manager else None, eval_fn)
    if writer is not None:
        writer.close()
    if dist.is_initialized():
        dist.destroy_process_group()
    return result


if __name__ == '__main__':
    app.run(main)

"""The 48-flag surface of the reference's `tf2/run.py:37-238` (names, types,
defaults and enums identical), plus the engine flags of this implementation.

As in the reference, layers read the process-global `FLAGS` at construction
(`tf2/model.py:160-170,234-238`, `tf2/resnet.py:50,330,400,442,566`).  The
TPU/GCP flags parse but are inert.
"""
from absl import flags

FLAGS = flags.FLAGS

_DEFINED = False


def define_flags():
    global _DEFINED
    if _DEFINED or 'learning_rate' in flags.FLAGS:
        _DEFINED = True
        return
    _DEFINED = True
    f = flags
    f.DEFINE_float('learning_rate', 0.3, 'Initial learning rate per batch size of 256.')
    f.DEFINE_enum('learning_rate_scaling', 'linear', ['linear', 'sqrt'],
                  'How to scale the learning rate as a function of batch size.')
    f.DEFINE_float('warmup_epochs', 10, 'Number of epochs of warmup.')
    f.DEFINE_float('weight_decay', 1e-6, 'Amount of weight decay to use.')
    f.DEFINE_float('batch_norm_decay', 0.9, 'Batch norm decay parameter.')
    f.DEFINE_integer('train_batch_size', 512, 'Batch size for training.')
    f.DEFINE_string('train_split', 'train', 'Split for training.')
    f.DEFINE_integer('train_epochs', 100, 'Number of epochs to train for.')
    f.DEFINE_integer('train_steps', 0,
                     'Number of steps to train for. If provided, overrides train_epochs.')
    f.DEFINE_integer('eval_steps', 0,
                     'Number of steps to eval for. If not provided, evals over entire dataset.')
    f.DEFINE_integer('eval_batch_size', 256, 'Batch size for eval.')
    f.DEFINE_integer('checkpoint_epochs', 1, 'Number of epochs between checkpoints/summaries.')
    f.DEFINE_integer('checkpoint_steps', 0,
                     'Number of steps between checkpoints/summaries. If provided, overrides '
                     'checkpoint_epochs.')
    f.DEFINE_string('eval_split', 'validation', 'Split for evaluation.')
    f.DEFINE_string('dataset', 'imagenet2012', 'Name of a dataset.')
    f.DEFINE_bool('cache_dataset', False, 'Whether to cache the entire dataset in memory.')
    f.DEFINE_enum('mode', 'train', ['train', 'eval', 'train_then_eval'],
                  'Whether to perform training or evaluation.')
    f.DEFINE_enum('train_mode', 'pretrain', ['pretrain', 'finetune'],
                  'The train mode controls different objectives and trainable components.')
    f.DEFINE_bool('lineareval_while_pretraining', True,
                  'Whether to finetune supervised head while pretraining.')
    f.DEFINE_string('checkpoint', None,
                    'Loading from the given checkpoint for fine-tuning if a finetuning '
                    'checkpoint does not already exist in model_dir.')
    f.DEFINE_bool('zero_init_logits_layer', False,
                  'If True, zero initialize layers after avg_pool for supervised learning.')
    f.DEFINE_integer('fine_tune_after_block', -1,
                     'The layers after which block that we will fine-tune. -1 means fine-tuning '
                     'everything. 0 means fine-tuning after stem block. 4 means fine-tuning '
                     'just the linear head.')
    f.DEFINE_string('master', None, 'Address/name of the TensorFlow master to use (inert).')
    f.DEFINE_string('model_dir', None, 'Model directory for training.')
    f.DEFINE_string('data_dir', None, 'Directory where dataset is stored.')
    f.DEFINE_bool('use_tpu', True, 'Whether to run on TPU (inert: this implementation runs on H100).')
    f.DEFINE_string('tpu_name', None, 'The Cloud TPU to use for training (inert).')
    f.DEFINE_string('tpu_zone', None, '[Optional] GCE zone of the Cloud TPU (inert).')
    f.DEFINE_string('gcp_project', None, '[Optional] Project name for the Cloud TPU (inert).')
    f.DEFINE_enum('optimizer', 'lars', ['momentum', 'adam', 'lars'], 'Optimizer to use.')
    f.DEFINE_float('momentum', 0.9, 'Momentum parameter.')
    f.DEFINE_string('eval_name', None, 'Name for eval.')
    f.DEFINE_integer('keep_checkpoint_max', 5, 'Maximum number of checkpoints to keep.')
    f.DEFINE_integer('keep_hub_module_max', 1, 'Maximum number of Hub modules to keep.')
    f.DEFINE_float('temperature', 0.1, 'Temperature parameter for contrastive loss.')
    f.DEFINE_boolean('hidden_norm', True, 'Temperature parameter for contrastive loss.')
    f.DEFINE_enum('proj_head_mode', 'nonlinear', ['none', 'linear', 'nonlinear'],
                  'How the head projection is done.')
    f.DEFINE_integer('proj_out_dim', 128, 'Number of head projection dimension.')
    f.DEFINE_integer('num_proj_layers', 3, 'Number of non-linear head layers.')
    f.DEFINE_integer('ft_proj_selector', 0,
                     'Which layer of the projection head to use during fine-tuning. '
                     '0 means no projection head, and -1 means the final layer.')
    f.DEFINE_boolean('global_bn', True,
                     'Whether to aggregate BN statistics across distributed cores.')
    f.DEFINE_integer('width_multiplier', 1, 'Multiplier to change width of network.')
    f.DEFINE_integer('resnet_depth', 50, 'Depth of ResNet.')
    f.DEFINE_float('sk_ratio', 0., 'If it is bigger than 0, it will enable SK. Recommendation: 0.0625.')
    f.DEFINE_float('se_ratio', 0., 'If it is bigger than 0, it will enable SE.')
    f.DEFINE_integer('image_size', 224, 'Input image size.')
    f.DEFINE_float('color_jitter_strength', 1.0, 'The strength of color jittering.')
    f.DEFINE_boolean('use_blur', True, 'Whether or not to use Gaussian blur for augmentation during pretraining.')
    # ---- engine flags (not in the reference) ----
    f.DEFINE_enum('b200_precision', 'bf16', ['bf16', 'fp32'],
                  'Activation/operand storage type of the conv stack: bf16 (wgmma bf16, '
                  'fp32 accumulate) or fp32 (parity mode).')
    f.DEFINE_enum('b200_conv_engine', 'tc', ['tc', 'tc3', 'simt'],
                  'tc: wgmma/TMA implicit GEMM (default). tc3: three-way split-bf16 products on the wgmma engine '
                  '(fp32 storage, fp32-accurate: the tensor-core verification mode). '
                  'simt: CUDA-core fp32 verification engine.')
    f.DEFINE_enum('b200_jpeg_decode', 'host', ['host', 'device'],
                  'Where data.TFRecordBuilder decodes JPEGs: host (Pillow on a thread pool) or device (sm_90a '
                  'kernels, bit-exact with Pillow; other formats and unsupported JPEGs stay on the host).')
    f.DEFINE_boolean('b200_fold_bn', False,
                     'Inference-mode forwards (evaluation, frozen block groups and stem when fine-tuning, the '
                     'distillation teacher) fold each BatchNorm on its moving statistics into the preceding conv or '
                     'dense layer: one launch writes the BatchNorm (+ residual, + ReLU) output.  bf16 on the tc engine '
                     'only.')
    f.DEFINE_integer('b200_num_classes', 1000, 'Classes of the supervised head when no dataset is read.')
    f.DEFINE_integer('b200_num_examples', 1281167, 'Examples per epoch when no dataset is read.')
    f.DEFINE_integer('b200_num_eval_examples', 50000, 'Evaluation examples when no dataset is read.')
    # SimCLRv2 distillation (distill.py): a frozen teacher's temperature-softened predictions train the student
    f.DEFINE_string('b200_distill_teacher', None,
                    'Teacher weights for distillation: a ckpt-N.npz, a TensorFlow checkpoint prefix, or a directory '
                    '(its latest checkpoint).  With --train_mode=finetune the training loss becomes distillation '
                    '(labels are not used); not allowed with --train_mode=pretrain.')
    f.DEFINE_float('b200_distill_temperature', 1.0, 'Distillation temperature T.')
    f.DEFINE_integer('b200_teacher_resnet_depth', None, 'Teacher resnet_depth (None: the student\'s).')
    f.DEFINE_integer('b200_teacher_width_multiplier', None, 'Teacher width_multiplier (None: the student\'s).')
    f.DEFINE_float('b200_teacher_sk_ratio', None, 'Teacher sk_ratio (None: the student\'s).')
    f.DEFINE_float('b200_teacher_se_ratio', None, 'Teacher se_ratio (None: the student\'s).')
    f.DEFINE_integer('b200_teacher_ft_proj_selector', None, 'Teacher ft_proj_selector (None: the student\'s).')
    # Generalized contrastive loss (Chen, Luo, Li 2021; objective.generalized_contrastive_forward)
    f.DEFINE_enum('b200_gcl_dist', 'none', ['none', 'logsumexp', 'normal', 'uniform'],
                  'Pretraining objective: none is NT-Xent; otherwise the generalized contrastive loss with this '
                  'distribution term: logsumexp (decoupled NT-Xent), or the sliced Wasserstein distance to a normal '
                  'or uniform prior.  It uses --temperature (the colab\'s default is 1.0, this flag\'s 0.1) and '
                  '--hidden_norm.  Only with --train_mode=pretrain.')
    f.DEFINE_float('b200_gcl_lambda', 1.0, 'Weight of the distribution term of the generalized contrastive loss.')
    f.DEFINE_float('b200_gcl_loss_scaling', 1.0, 'Scale of the generalized contrastive loss.')


define_flags()

REFERENCE_FLAG_NAMES = [
    'learning_rate', 'learning_rate_scaling', 'warmup_epochs', 'weight_decay', 'batch_norm_decay',
    'train_batch_size', 'train_split', 'train_epochs', 'train_steps', 'eval_steps', 'eval_batch_size',
    'checkpoint_epochs', 'checkpoint_steps', 'eval_split', 'dataset', 'cache_dataset', 'mode',
    'train_mode', 'lineareval_while_pretraining', 'checkpoint', 'zero_init_logits_layer',
    'fine_tune_after_block', 'master', 'model_dir', 'data_dir', 'use_tpu', 'tpu_name', 'tpu_zone',
    'gcp_project', 'optimizer', 'momentum', 'eval_name', 'keep_checkpoint_max', 'keep_hub_module_max',
    'temperature', 'hidden_norm', 'proj_head_mode', 'proj_out_dim', 'num_proj_layers',
    'ft_proj_selector', 'global_bn', 'width_multiplier', 'resnet_depth', 'sk_ratio', 'se_ratio',
    'image_size', 'color_jitter_strength', 'use_blur',
]


def set_flags(**kw):
    """Programmatic flag assignment for tests / bench (marks FLAGS parsed)."""
    if not FLAGS.is_parsed():
        FLAGS(['simclr_b200'])
    for k, v in kw.items():
        setattr(FLAGS, k, v)

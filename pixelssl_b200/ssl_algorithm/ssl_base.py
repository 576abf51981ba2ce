"""The algorithm contract of pixelssl/ssl_algorithm/ssl_base.py:19-159: module-level
``add_parser_arguments(parser)``, an export function named like the module, and an object with
``build / train / validate / save_checkpoint / load_checkpoint`` plus ``NAME`` and
``SUPPORTED_TASK_TYPES``.  TaskProxy (task_template/proxy.py:134-159,433-441) only ever touches
these."""
import os
import time

import torch

from ..utils import logger, tool
from ..task.sseg import evaluation


def add_parser_arguments(parser):
    pass


class _SSLBase:
    NAME = 'ssl_base'
    SUPPORTED_TASK_TYPES = []
    RAMPUP_EPOCHS = None         # name of the ramp-up argument (e.g. 'cons_rampup_epochs'); None: total_steps = 0
    LOG_LINES = ''               # the step log line after the shared 'step: ... batch-time: ...' line
    ITER_LRERS = ()              # keys of self.lrers stepped every iteration whatever is_epoch_lrer says
    VALIDATION_IDS = ('task',)   # the id_str of every _metrics call of validate_step

    def __init__(self, args):
        self.args = args
        self.task_func = None
        self.meters = logger.AvgMeterSet()
        self.models, self.optimizers, self.lrers, self.criterions = {}, {}, {}, {}

    def build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        evaluation.check_args(self.args)
        self._build(model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func)

    def train(self, data_loader, epoch):
        self._train(data_loader, epoch)
        self._flush_log()

    def validate(self, data_loader, epoch):
        """``_validate`` inside the multi-view evaluation scope: an eval-mode task model then forwards the views of
        ``--val-protocol`` / ``--val-scales`` / ``--val-flip`` (task/sseg/evaluation.py); the default protocol changes
        nothing."""
        self._flush_log()
        with evaluation.validating():
            self._validate(data_loader, epoch)

    def _log_step(self, make_line):
        """The per-step log line of every reference ``_train`` (e.g. ssl_mt.py:199-207), emitted ONE logging
        interval late: formatting the meters right away is a device->host read that drains the launch queue every
        ``log_freq`` steps (at log_freq = 1 the GPU idles while the host re-fills it).  The meter values of this
        step are copied to pinned host memory asynchronously now and printed at the next call / at the end of
        ``train()``, by which time the copy has long completed.  Same text, same values."""
        snap = self.meters.snapshot()
        prev, self._pending_log = getattr(self, '_pending_log', None), (make_line, snap)
        if prev is not None:
            logger.log_info(prev[0](prev[1]))

    def _flush_log(self):
        prev, self._pending_log = getattr(self, '_pending_log', None), None
        if prev is not None:
            logger.log_info(prev[0](prev[1]))

    def save_checkpoint(self, epoch):
        """``{'algorithm', 'epoch'}`` plus the state dict of every model, optimizer and lr scheduler under its key
        in ``self.models`` / ``self.optimizers`` / ``self.lrers``: the reference's checkpoint layout
        (e.g. ssl_mt.py:296-307)."""
        state = {'algorithm': self.NAME, 'epoch': epoch}
        for elements in (self.models, self.optimizers, self.lrers):
            state.update((key, element.state_dict()) for key, element in elements.items())
        torch.save(state, os.path.join(self.args.checkpoint_path, 'checkpoint_{0}.ckpt'.format(epoch)))

    def load_checkpoint(self):
        """Loads ``args.resume`` into every model, optimizer and lr scheduler; the loaded momentum buffers / Adam
        moments of optimizer ``x_optimizer`` move into the parameter arena of model ``x_model``.  Returns the
        epoch."""
        checkpoint = torch.load(self.args.resume, weights_only=False)
        name = tool.dict_value(checkpoint, 'algorithm', default='unknown')
        if name != self.NAME:
            logger.log_err('Unmatched SSL algorithm format in checkpoint => required: {0} - given: {1}\n'
                           .format(self.NAME, name))
        for key, model in self.models.items():
            model.load_state_dict(checkpoint[key])
        for key, optimizer in self.optimizers.items():
            optimizer.load_state_dict(checkpoint[key])
            self.models[key.replace('optimizer', 'model')].arena.adopt_optimizer_state(optimizer)
        for key, lrer in self.lrers.items():
            lrer.load_state_dict(checkpoint[key])
        return checkpoint['epoch']

    def _train(self, data_loader, epoch):
        """One epoch of every reference ``_train`` (e.g. ssl_mt.py:124-224): ``train_step`` per batch, timed, a step
        log line every ``log_freq`` steps and the lr schedulers stepped per iteration or per epoch."""
        self.meters.reset()
        for model in self.models.values():
            model.train()
        rampup_epochs = getattr(self.args, self.RAMPUP_EPOCHS) if self.RAMPUP_EPOCHS else 0
        line = 'step: [{0}][{1}/{2}]\tbatch-time: {meters[batch_time]:.3f}\n' + self.LOG_LINES
        for idx, (inp, gt) in enumerate(device_prefetch(data_loader)):
            timer = time.time()
            cur_step = len(data_loader) * epoch + idx
            total_steps = len(data_loader) * rampup_epochs
            self.train_step(inp, gt, cur_step, total_steps)
            self.meters.update('batch_time', time.time() - timer)
            if idx % self.args.log_freq == 0:
                self._log_step(lambda m, a=(epoch + 1, idx, len(data_loader), self.args.task): line.format(*a, meters=m))
            for key, lrer in self.lrers.items():
                if key in self.ITER_LRERS or not self.args.is_epoch_lrer:
                    lrer.step()
        if self.args.is_epoch_lrer:
            for key, lrer in self.lrers.items():
                if key not in self.ITER_LRERS:
                    lrer.step()

    def _validate(self, data_loader, epoch):
        """Every reference ``_validate`` (e.g. ssl_mt.py:226-294): eval mode, ``validate_step`` per batch, then the
        'Validation metrics' summary."""
        self.meters.reset()
        for model in self.models.values():
            model.eval()
        for inp, gt in data_loader:
            self.validate_step(inp, gt)
        self._log_validation_metrics(self.VALIDATION_IDS)

    def _validate_model(self, model, criterion, inp, gt, meter, id_str):
        """The validation body of one task model: forward, mean task loss into ``meter``, metrics under ``id_str``."""
        resulter, _ = model.forward(inp)
        pred = tool.dict_value(resulter, 'pred')
        self.meters.update(meter, torch.mean(criterion.forward(pred, gt, inp)).data)
        self._metrics(resulter, gt, inp, id_str)

    def _metrics(self, resulter, gt, inp, id_str):
        """``self.task_func.metrics(activated_pred, gt, inp, self.meters, id_str=...)`` of every
        reference ``_validate`` (e.g. ssl_mt.py:264-265, ssl_null.py:169)."""
        if self.task_func is None or not hasattr(self.task_func, 'metrics'):
            return
        activated_pred = resulter.get('activated_pred') if resulter is not None else None
        if activated_pred is None:
            self._pred_err()
        self.task_func.metrics(activated_pred, gt, inp, self.meters, id_str=id_str)

    def _log_validation_metrics(self, id_strs):
        """The 'Validation metrics' epilogue of every reference ``_validate`` (ssl_mt.py:285-294)."""
        if self.task_func is None or not hasattr(self.task_func, 'METRIC_STR'):
            return
        info = {i: '' for i in id_strs}
        for key in sorted(list(self.meters.keys())):
            if self.task_func.METRIC_STR in key:
                for id_str in info:
                    if key.startswith(id_str):
                        info[id_str] += '{0}: {1:.6}\t'.format(key, self.meters[key])
        logger.log_info('Validation metrics:\n' + ''.join(
            '  {0}-metrics\t=>\t{1}\n'.format(i, info[i].replace('_', '-')) for i in id_strs))

    def _pred_err(self):
        logger.log_err('In {0}, the \'resulter\' dict returned by the task model should contain the following keys:\n'
                       '   (1) \'pred\'\t=>\tunactivated task predictions\n'
                       '   (2) \'activated_pred\'\t=>\tactivated task predictions\n'.format(self.NAME.upper()))

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        raise NotImplementedError

    def train_step(self, inp, gt, cur_step, total_steps):
        raise NotImplementedError

    def validate_step(self, inp, gt):
        raise NotImplementedError


_prefetch_state = {}


def device_prefetch(data_loader):
    """Iterate ``data_loader`` one batch ahead: the host->HBM copy of batch k+1 (``Variable(i).cuda()`` of the
    reference's ``_batch_prehandle``, e.g. ssl_mt.py:337-357) is enqueued on a side stream before step k's kernels
    are, so it overlaps the compute instead of sitting in front of it.  Yields ``(inp, gt)`` tuples of DEVICE
    tensors (``to_device`` then passes them through); falls back to plain iteration without CUDA.

    The device side is two fixed staging slots (allocated once per tensor shape): slot k % 2 is rewritten only after
    the step that consumed it has finished, so no allocator traffic (and no cudaMalloc stall) sits in the loop.  A
    yielded batch is valid until the iteration after next."""
    if not torch.cuda.is_available():
        for batch in data_loader:
            yield batch
        return
    # the copy stream, the staging slots and their "consumed" events live as long as the process: a new side stream per
    # epoch gets no cached blocks from torch's (per-stream) allocator pools, and a cudaMalloc of the 67 MB slots at the
    # start of an epoch stalls the step
    state = _prefetch_state.get(torch.cuda.current_device())
    if state is None:
        state = _prefetch_state[torch.cuda.current_device()] = {
            'stream': torch.cuda.Stream(), 'slots': [{}, {}], 'done': [None, None]}
    copy_stream = state['stream']
    slots = state['slots']           # slot -> {(position, shape, dtype): device tensor}
    done = state['done']             # event on the main stream: the step that read this slot is enqueued

    def stage(batch, k):
        inp, gt = batch
        b = k % 2
        if done[b] is not None:
            copy_stream.wait_event(done[b])
        out = []
        with torch.cuda.stream(copy_stream):
            for pos, t in enumerate(tuple(inp) + tuple(gt)):
                if t.is_cuda:
                    out.append(t)
                    continue
                key = (pos, tuple(t.shape), t.dtype)
                buf = slots[b].get(key)
                if buf is None:
                    buf = slots[b][key] = torch.empty(t.shape, dtype=t.dtype, device='cuda')
                buf.copy_(t, non_blocking=True)
                out.append(buf)
        ev = torch.cuda.Event()
        ev.record(copy_stream)
        return tuple(out[:len(inp)]), tuple(out[len(inp):]), ev

    it = iter(data_loader)
    try:
        nxt = stage(next(it), 0)
    except StopIteration:
        return
    k = 0
    while nxt is not None:
        cur = nxt
        try:
            nxt = stage(next(it), k + 1)
        except StopIteration:
            nxt = None
        main = torch.cuda.current_stream()
        main.wait_event(cur[2])
        yield cur[0], cur[1]
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        done[k % 2] = ev
        k += 1


def to_device(tensors, non_blocking=True):
    """``Variable(i).cuda()`` of every ``_batch_prehandle`` (ssl_mt.py:337-357): host -> HBM copy on
    the current stream (asynchronous when the loader pinned the batch)."""
    return tuple(t.cuda(non_blocking=non_blocking) for t in tensors)


def pair_picker(name, model_dict, optimizer_dict, lrer_dict, criterion_dict):
    """The element dicts of an algorithm that trains two task models side by side (ssl_gct.py:31-48): one entry
    ``model`` serves both sides, or two entries ``lmodel`` / ``rmodel``.  Returns ``pick(d) -> [left, right]``."""
    tag = name.upper()
    if not len(model_dict) == len(optimizer_dict) == len(lrer_dict) == len(criterion_dict):
        logger.log_err('The len(element_dict) of {0} should be the same\n'.format(tag))
    if len(model_dict) == 1:
        if list(model_dict.keys())[0] != 'model':
            logger.log_err('In {0}, the key of 1-value element_dict should be \'model\',\n'
                           'but \'{1}\' is given\n'.format(tag, model_dict.keys()))
        return lambda d: [d['model'], d['model']]
    if len(model_dict) == 2:
        if 'lmodel' not in model_dict or 'rmodel' not in model_dict:
            logger.log_err('In {0}, the key of 2-value element_dict should be \'(lmodel, rmodel)\', '
                           'but \'{1}\' is given\n'.format(tag, model_dict.keys()))
        return lambda d: [d['lmodel'], d['rmodel']]
    logger.log_err('The {0} algorithm supports element_dict with 1 or 2 elements, '
                   'but given {1} elements\n'.format(tag, len(model_dict)))


def check_single_model_dicts(name, model_dict, optimizer_dict, lrer_dict, criterion_dict):
    if not len(model_dict) == len(optimizer_dict) == len(lrer_dict) == len(criterion_dict) == 1:
        logger.log_err('The len(element_dict) of {0} should be 1\n'.format(name.upper()))
    elif list(model_dict.keys())[0] != 'model':
        logger.log_err('In {0}, the key of element_dict should be \'model\',\n'
                       'but \'{1}\' is given\n'.format(name.upper(), model_dict.keys()))

"""`mx.callback.Speedometer` and `mx.callback.module_checkpoint` (SNIPER-mxnet/python/mxnet/callback.py:27-52, 120-170)
for Trainer.fit.  With several ranks only rank 0 logs and writes files; every rank still reads the metrics, because
that read is a collective."""
import logging
import time

import torch


def _rank0():
    return not (torch.distributed.is_available() and torch.distributed.is_initialized()) or \
        torch.distributed.get_rank() == 0


class Speedometer(object):
    """Logs the speed and the metrics every `frequent` batches: `Epoch[%d] Batch [%d]\\tSpeed: %.2f samples/sec` and
    `\\t%s=%f` per metric, resetting the metrics after each print when auto_reset.  The first call of an epoch (a batch
    count lower than the last one) only starts the clock."""

    def __init__(self, batch_size, frequent=50, auto_reset=True):
        self.batch_size = batch_size
        self.frequent = frequent
        self.init = False
        self.tic = 0
        self.last_count = 0
        self.auto_reset = auto_reset

    def __call__(self, param):
        count = param.nbatch
        if self.last_count > count:
            self.init = False
        self.last_count = count

        if self.init:
            if count % self.frequent == 0:
                speed = self.frequent * self.batch_size / (time.time() - self.tic)
                if param.eval_metric is not None:
                    name_value = param.eval_metric.get_name_value()
                    if self.auto_reset:
                        param.eval_metric.reset()
                    if _rank0():
                        msg = 'Epoch[%d] Batch [%d]\tSpeed: %.2f samples/sec'
                        msg += '\t%s=%f' * len(name_value)
                        logging.info(msg, param.epoch, count, speed, *sum(name_value, ()))
                elif _rank0():
                    logging.info("Iter[%d] Batch [%d]\tSpeed: %.2f samples/sec", param.epoch, count, speed)
                self.tic = time.time()
        else:
            self.init = True
            self.tic = time.time()


def module_checkpoint(trainer, prefix, period=1, save_optimizer_states=True):
    """Epoch-end callback: every `period` epochs, `<prefix>-%04d.params` for epoch + 1 (with the `*_test` tensors of
    checkpoint_callback), `<prefix>-symbol.json` when the net was bound from a Symbol, and with save_optimizer_states
    `<prefix>-%04d.states` (Trainer.save_checkpoint), from the arg / aux params fit passes."""
    period = int(max(1, period))

    def _callback(iter_no, sym=None, arg=None, aux=None):
        if (iter_no + 1) % period == 0 and _rank0():
            # arg / aux: what fit exported on every rank (moving statistics averaged over the ranks)
            trainer.save_checkpoint(prefix, iter_no + 1, save_optimizer_states, arg_params=arg, aux_params=aux)
    return _callback

"""Learning-rate schedules of the SVB generator optimizer (reference: utils/common_schedulers.py).  Each sets the lr of every param
group of its optimizer in ``step(num_updates)``; the task calls ``step(global_step)`` after each generator update."""
from neuralsvb_b200.utils.hparams import hparams


class NoneSchedule:
    """Constant ``hparams['lr']``."""

    def __init__(self, optimizer):
        self.optimizer = optimizer
        self.constant_lr = hparams['lr']
        self.step(0)

    def step(self, num_updates):
        self.lr = self.constant_lr
        for param_group in self.optimizer.param_groups:
            param_group['lr'] = self.lr
        return self.lr

    def get_lr(self):
        return self.optimizer.param_groups[0]['lr']

    def get_last_lr(self):
        return self.get_lr()


class RSQRTSchedule(NoneSchedule):
    """Linear warm-up over ``warmup_updates``, then inverse square-root decay, scaled by ``hidden_size ** -0.5``; at least 1e-7:
    lr = max(lr * min(n / warmup, 1) * max(warmup, n) ** -0.5 * hidden_size ** -0.5, 1e-7)."""

    def __init__(self, optimizer):
        self.warmup_updates = hparams['warmup_updates']
        self.hidden_size = hparams['hidden_size']
        super().__init__(optimizer)

    def step(self, num_updates):
        warmup = min(num_updates / self.warmup_updates, 1.0)
        rsqrt_decay = max(self.warmup_updates, num_updates) ** -0.5
        self.lr = max(self.constant_lr * warmup * rsqrt_decay * self.hidden_size ** -0.5, 1e-7)
        for param_group in self.optimizer.param_groups:
            param_group['lr'] = self.lr
        return self.lr

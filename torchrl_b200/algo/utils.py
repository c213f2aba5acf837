"""Small algorithm helpers (API of /root/reference/torchrl/algo/utils.py:5-32).  Cold-path torch statements: the
agents use the fused kernels (trl_qr_dqn_loss, trl_polyak_update) on their flat buffers instead."""
import torch


def four_stats(prefix, values):
    """{prefix/mean, prefix/std, prefix/max, prefix/min} from four values in that order (an info-row slice written by
    ops.vec_stats, or four 0-d tensors)."""
    return {prefix + "/" + s: float(v) for s, v in zip(("mean", "std", "max", "min"), values)}


def huber(x, k=1.0):
    """0.5 x^2 inside |x| < k, k (|x| - k/2) outside."""
    magnitude = x.abs()
    return torch.where(magnitude < k, 0.5 * x * x, k * (magnitude - 0.5 * k))


def quantile_regression_loss(coefficient, source, target):
    """mean over (batch, target quantile j, source quantile i) of huber(t_j - s_i) * |tau_i - [t_j - s_i < 0]|
    (utils.py:5-9)."""
    gap = target[..., :, None] - source[..., None, :]
    below = (gap.detach() < 0).float()
    return (huber(gap) * (coefficient - below).abs()).mean()


def _pairs(source, target):
    return zip(target.parameters(), source.parameters())


def soft_update_from_to(source, target, tau):
    """theta' <- (1 - tau) theta' + tau theta, tensor by tensor (both products rounded before the sum, like the
    reference's expression)."""
    with torch.no_grad():
        for theta_t, theta in _pairs(source, target):
            torch.add(theta_t.data * (1.0 - tau), theta.data * tau, out=theta_t.data)


def copy_model_params_from_to(source, target):
    with torch.no_grad():
        for theta_t, theta in _pairs(source, target):
            theta_t.data.copy_(theta.data)


def update_linear_schedule(optimizer, epoch, total_num_epochs, initial_lr):
    """lr(epoch) = initial_lr * (1 - epoch / total) written to every param group (utils.py:28-32)."""
    lr = initial_lr - (initial_lr * (epoch / float(total_num_epochs)))
    for group in optimizer.param_groups:
        group['lr'] = lr

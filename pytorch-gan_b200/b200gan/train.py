"""Training steps of the hot-path scripts, re-enacted around the drop-in modules, plus the CUDA-graph
runner used by bench.py.  The step bodies follow the reference loops line by line so that the
unmodified scripts (via launch.py) and this module execute the same sequence of operator calls.
"""
import contextlib

import torch

from . import ops


@contextlib.contextmanager
def frozen(module):
    """Temporarily mark a network's parameters as not requiring grad.  The reference back-propagates the
    generator loss into the discriminator's weights too (dcgan.py:168) and throws those gradients away at
    optimizer_D.zero_grad() (dcgan.py:175); skipping that dead weight-gradient work changes no result."""
    params = [p for p in module.parameters() if p.requires_grad]
    for p in params:
        p.requires_grad_(False)
    try:
        yield
    finally:
        for p in params:
            p.requires_grad_(True)


def _opt_step(opt, reducer):
    """optimizer.step(), preceded by the data-parallel gradient all-reduce when a reducer is given (ddp.py)."""
    if reducer is None:
        opt.step()
    elif hasattr(reducer, "reduce_and_step"):
        reducer.reduce_and_step(opt)
    else:
        reducer()
        opt.step()


def _join(*reducers):
    for r in reducers:
        if r is not None and hasattr(r, "join"):
            r.join()


def _d_passes_batchable(discriminator, real_imgs, loss):
    """The two discriminator passes of the D step can run as one grouped pass: a DCGAN-style module (`model` = conv blocks
    that the fused chain covers completely, `adv_layer` without batch-dependent modules, zoo.DCGANDiscriminator /
    dcgan.py:73-99), a mean-reduced element-wise loss, training mode."""
    from . import nn as bnn
    if not getattr(discriminator, "_b200_batchable_passes", False):
        return False
    if not (discriminator.training and real_imgs.is_cuda and real_imgs.dim() == 4 and real_imgs.dtype == torch.float32):
        return False
    if not isinstance(loss, (torch.nn.BCELoss, torch.nn.MSELoss)) or loss.reduction != "mean":
        return False
    if getattr(loss, "weight", None) is not None:
        return False
    shape = (2 * real_imgs.shape[0],) + tuple(real_imgs.shape[1:])
    return bnn.groups_eligible(discriminator.model, shape, 2)


def dcgan_step(generator, discriminator, opt_g, opt_d, real_imgs, z, loss=None, valid=None, fake=None,
               reduce_g=None, reduce_d=None, skip_dead_wgrad=True):
    """implementations/dcgan/dcgan.py:146-183.  `reduce_*`: optional gradient all-reduce hooks invoked
    right before the corresponding optimizer step (data parallel, SURVEY.md section 8e)."""
    loss = loss or torch.nn.BCELoss()
    n = real_imgs.shape[0]
    if valid is None:
        valid = torch.ones(n, 1, device=real_imgs.device)   # dcgan.py:147
        fake = torch.zeros(n, 1, device=real_imgs.device)   # dcgan.py:148
    opt_g.zero_grad()                                        # :157
    gen_imgs = generator(z)                                  # :163
    with frozen(discriminator) if skip_dead_wgrad else contextlib.nullcontext():
        g_loss = loss(discriminator(gen_imgs), valid)        # :166
        g_loss.backward()                                    # :168
    _opt_step(opt_g, reduce_g)                               # :169 (all-reduce + Adam may overlap the D phase below)
    opt_d.zero_grad()                                        # :175
    if _d_passes_batchable(discriminator, real_imgs, loss):
        # :178-180 as ONE pass over [real; fake] with two BatchNorm statistics groups (ops.bn_groups): same batch
        # statistics, running-statistics updates, dropout masks and summed parameter gradients as the two passes, half the
        # launches.  mean over 2N outputs == (mean over real + mean over fake) / 2.
        with ops.bn_groups(2):
            out = discriminator(torch.cat([real_imgs, gen_imgs.detach()]))
        d_loss = loss(out, torch.cat([valid, fake]))
    else:
        real_loss = loss(discriminator(real_imgs), valid)        # :178
        fake_loss = loss(discriminator(gen_imgs.detach()), fake) # :179
        d_loss = (real_loss + fake_loss) / 2                     # :180
    d_loss.backward()                                        # :182
    _opt_step(opt_d, reduce_d)                               # :183
    _join(reduce_g, reduce_d)
    return g_loss.detach(), d_loss.detach(), gen_imgs.detach()


def gan_step(generator, discriminator, opt_g, opt_d, real_imgs, z, loss=None):
    """implementations/gan/gan.py:124-161, the vanilla MLP GAN: on the drop-in modules the generator runs on the fused
    MLP generator kernels and each discriminator pass on the critic kernels' Sigmoid mode (functional.MlpGeneratorFn,
    functional.MlpDiscriminatorFn).  D is frozen during the G step, as in dcgan_step."""
    loss = loss or torch.nn.BCELoss()
    n = real_imgs.shape[0]
    valid = torch.ones(n, 1, device=real_imgs.device)           # :125
    fake = torch.zeros(n, 1, device=real_imgs.device)           # :126
    opt_g.zero_grad()                                           # :135
    gen_imgs = generator(z)                                     # :141
    with frozen(discriminator):
        g_loss = loss(discriminator(gen_imgs), valid)           # :144
        g_loss.backward()                                       # :146
    opt_g.step()                                                # :147
    opt_d.zero_grad()                                           # :153
    real_loss = loss(discriminator(real_imgs), valid)           # :156
    fake_loss = loss(discriminator(gen_imgs.detach()), fake)    # :157
    d_loss = (real_loss + fake_loss) / 2                        # :158
    d_loss.backward()                                           # :160
    opt_d.step()                                                # :161
    return g_loss.detach(), d_loss.detach(), gen_imgs.detach()


def wgan_gp_critic_step(generator, discriminator, opt_d, real_imgs, z, alpha, lambda_gp=10.0, fused_gp=True,
                        reduce_d=None):
    """One critic iteration of implementations/wgan_gp/wgan_gp.py:155-174.  `alpha` [N,1,1,1] is the
    interpolation weight the reference draws with numpy (wgan_gp.py:122).  A truthy fused_gp (True or "step") runs
    the whole iteration -- three critic passes, the penalty and the backward -- in one cooperative kernel
    (functional.critic_step_mlp, MLP critic only); fused_gp=False builds the penalty with autograd exactly like the
    reference, which on the drop-in modules runs on the fused critic kernels.
    The reference leaves fake_imgs attached (dead back-prop into G, whose grads are zeroed at :176); here the
    fakes are detached -- identical D update."""
    from . import functional as F
    opt_d.zero_grad()                                                     # :155
    with torch.no_grad():
        fake_imgs = generator(z)                                          # :161
    if fused_gp:
        d_loss, gp_term = F.critic_step_mlp(discriminator.model, real_imgs, fake_imgs, alpha, lambda_gp)
        d_loss.backward()
        _opt_step(opt_d, reduce_d)
        _join(reduce_d)
        return d_loss.detach(), gp_term.detach()
    real_validity = discriminator(real_imgs)                              # :164
    fake_validity = discriminator(fake_imgs)                              # :166
    interpolates = alpha * real_imgs + (1 - alpha) * fake_imgs            # :124
    interpolates = interpolates.requires_grad_(True)
    d_int = discriminator(interpolates)                                   # :125
    grads = torch.autograd.grad(outputs=d_int, inputs=interpolates, grad_outputs=torch.ones_like(d_int),
                                create_graph=True, retain_graph=True, only_inputs=True)[0]   # :128-135
    grads = grads.view(grads.size(0), -1)
    gp_term = lambda_gp * ((grads.norm(2, dim=1) - 1) ** 2).mean()        # :137
    d_loss = -torch.mean(real_validity) + torch.mean(fake_validity) + gp_term   # :171
    d_loss.backward()                                                     # :173
    _opt_step(opt_d, reduce_d)                                            # :174
    _join(reduce_d)
    return d_loss.detach(), gp_term.detach()


def wgan_gp_generator_step(generator, discriminator, opt_g, z):
    """wgan_gp.py:176-193."""
    opt_g.zero_grad()
    with frozen(discriminator):
        g_loss = -torch.mean(discriminator(generator(z)))
        g_loss.backward()
    opt_g.step()
    return g_loss.detach()


def _built_from_dropins(*nets):
    from . import nn as bnn
    dropin = tuple(bnn.REPLACEMENTS.values())
    return any(isinstance(m, dropin) for net in nets for m in net.modules())


def _pixel_losses(*nets):
    """(mse, l1) for a translator's step: the drop-in MSELoss / L1Loss (csrc/pixel_loss) when the networks are built from
    drop-in modules, else torch's own functional losses, so that a stock model keeps every op on stock torch."""
    from . import nn as bnn
    if _built_from_dropins(*nets):
        return bnn.MSELoss(), bnn.L1Loss()
    return torch.nn.functional.mse_loss, torch.nn.functional.l1_loss


def acgan_step(generator, discriminator, opt_g, opt_d, real_imgs, labels, z, gen_labels):
    """implementations/acgan/acgan.py:184-223, with the noise z and the int64 class indices gen_labels drawn by the
    caller (:187-188).  BCELoss and CrossEntropyLoss (:112-113) are the drop-ins when the networks are built from
    drop-in modules, else torch's own.  D is frozen during the G step, as in dcgan_step.  Returns the two losses, the
    fakes and the class posteriors of the real and the fake pass (the script's accuracy readback, :218-220)."""
    from . import nn as bnn
    ns = bnn if _built_from_dropins(generator, discriminator) else torch.nn
    adversarial_loss, auxiliary_loss = ns.BCELoss(), ns.CrossEntropyLoss()
    n = real_imgs.shape[0]
    valid = torch.ones(n, 1, device=real_imgs.device)                                        # :173
    fake = torch.zeros(n, 1, device=real_imgs.device)                                        # :174
    opt_g.zero_grad()                                                                        # :184
    gen_imgs = generator(z, gen_labels)                                                      # :191
    with frozen(discriminator):
        validity, pred_label = discriminator(gen_imgs)                                       # :194
        g_loss = 0.5 * (adversarial_loss(validity, valid) + auxiliary_loss(pred_label, gen_labels))  # :195
        g_loss.backward()                                                                    # :197
    opt_g.step()                                                                             # :198
    opt_d.zero_grad()                                                                        # :204
    real_pred, real_aux = discriminator(real_imgs)                                           # :207
    d_real_loss = (adversarial_loss(real_pred, valid) + auxiliary_loss(real_aux, labels)) / 2           # :208
    fake_pred, fake_aux = discriminator(gen_imgs.detach())                                   # :211
    d_fake_loss = (adversarial_loss(fake_pred, fake) + auxiliary_loss(fake_aux, gen_labels)) / 2        # :212
    d_loss = (d_real_loss + d_fake_loss) / 2                                                 # :215
    d_loss.backward()                                                                        # :222
    opt_d.step()                                                                             # :223
    return g_loss.detach(), d_loss.detach(), gen_imgs.detach(), real_aux.detach(), fake_aux.detach()


def pix2pix_step(generator, discriminator, opt_g, opt_d, real_a, real_b, lambda_pixel=100.0, reduce_g=None,
                 reduce_d=None):
    """implementations/pix2pix/pix2pix.py:131-172 (MSE GAN loss :50, L1 pixel loss :51,:54)."""
    mse, l1 = _pixel_losses(generator, discriminator)
    opt_g.zero_grad()                                          # :138
    fake_b = generator(real_a)                                 # :141
    with frozen(discriminator):
        pred_fake = discriminator(fake_b, real_a)              # :142
        valid = torch.ones_like(pred_fake)                     # :131
        loss_g = mse(pred_fake, valid) + lambda_pixel * l1(fake_b, real_b)   # :143-148
        loss_g.backward()                                      # :150
    _opt_step(opt_g, reduce_g)                                 # :152
    opt_d.zero_grad()                                          # :158
    loss_real = mse(discriminator(real_b, real_a), valid)      # :161-162
    loss_fake = mse(discriminator(fake_b.detach(), real_a), torch.zeros_like(valid))   # :165-166
    loss_d = 0.5 * (loss_real + loss_fake)                     # :169
    loss_d.backward()                                          # :171
    _opt_step(opt_d, reduce_d)                                 # :172
    _join(reduce_g, reduce_d)
    return loss_g.detach(), loss_d.detach()


class ReplayBuffer:
    """History of generated images (cyclegan/utils.py:13-33): each incoming sample is either passed through or
    swapped with a stored one (python `random`, per sample) -- index bookkeeping only, bit-exact."""

    def __init__(self, max_size=50):
        assert max_size > 0
        self.max_size, self.data = max_size, []

    def push_and_pop(self, data):
        import random
        out = []
        for element in data.detach():
            element = element.unsqueeze(0)
            if len(self.data) < self.max_size:
                self.data.append(element)
                out.append(element)
            elif random.uniform(0, 1) > 0.5:
                i = random.randint(0, self.max_size - 1)
                out.append(self.data[i].clone())
                self.data[i] = element
            else:
                out.append(element)
        return torch.cat(out)


def cyclegan_step(g_ab, g_ba, d_a, d_b, opt_g, opt_d_a, opt_d_b, real_a, real_b, buf_a=None, buf_b=None,
                  lambda_cyc=10.0, lambda_id=5.0, reduce_g=None, reduce_d_a=None, reduce_d_b=None):
    """implementations/cyclegan/cyclegan.py:163-241: 6 generator passes + 2 D passes for the G loss, then one
    step per discriminator on (real, replayed fake).  buf_* = ReplayBuffer or None (fakes used directly)."""
    mse, l1 = _pixel_losses(g_ab, g_ba, d_a, d_b)
    opt_g.zero_grad()                                                          # :177
    loss_identity = (l1(g_ba(real_a), real_a) + l1(g_ab(real_b), real_b)) / 2  # :180-183
    fake_b = g_ab(real_a)                                                      # :186
    fake_a = g_ba(real_b)                                                      # :188
    with frozen(d_a), frozen(d_b):
        pred_b, pred_a = d_b(fake_b), d_a(fake_a)
        valid = torch.ones_like(pred_b)                                        # :166
        loss_gan = (mse(pred_b, valid) + mse(pred_a, valid)) / 2               # :187-191
        loss_cycle = (l1(g_ba(fake_b), real_a) + l1(g_ab(fake_a), real_b)) / 2  # :194-199
        loss_g = loss_gan + lambda_cyc * loss_cycle + lambda_id * loss_identity  # :202
        loss_g.backward()                                                      # :204
    _opt_step(opt_g, reduce_g)                                                 # :205
    fake = torch.zeros_like(valid)                                             # :167
    losses_d = []
    for d, opt, real, fk, buf, red in ((d_a, opt_d_a, real_a, fake_a, buf_a, reduce_d_a),
                                       (d_b, opt_d_b, real_b, fake_b, buf_b, reduce_d_b)):
        opt.zero_grad()                                                        # :211 / :228
        fk_ = buf.push_and_pop(fk) if buf is not None else fk.detach()         # :216 / :233
        loss_d = (mse(d(real), valid) + mse(d(fk_.detach()), fake)) / 2        # :214-219
        loss_d.backward()                                                      # :221
        _opt_step(opt, red)                                                    # :222
        losses_d.append(loss_d.detach())
    _join(reduce_g, reduce_d_a, reduce_d_b)
    return loss_g.detach(), (losses_d[0] + losses_d[1]) / 2


class GraphedStep:
    """Capture one training step into a CUDA graph (static input/output buffers) and replay it.
    The step function must be free of host synchronisation; optimizers must be `capturable`."""

    def __init__(self, step_fn, example_inputs, warmup=3):
        self.static_in = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self.static_out = step_fn(*self.static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_out = step_fn(*self.static_in)

    def __call__(self, *inputs):
        for s, t in zip(self.static_in, inputs):
            s.copy_(t, non_blocking=True)
        self.graph.replay()
        return self.static_out

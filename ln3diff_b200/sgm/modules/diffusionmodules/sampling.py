"""Mirror of reference sgm/modules/diffusionmodules/sampling.py:21-362 (the sgm sampler family).

`EulerEDMSampler(...)(denoiser, x, cond, uc)` keeps the reference loop.  The per-step elementwise
tail -- VanillaCFG combine (guiders.py:28-31), to_d (sampling_utils.py:34-35) and the Euler step
(sampling.py:78-79) -- is one ln3_sampler_affine_update launch on CUDA tensors:
    x' = (1 + dt/s) x - (dt/s)(1 - g) D_u - (dt/s) g D_c,   dt = s_next - s, g = cfg scale.

HeunEDMSampler, EulerAncestralSampler, DPMPP2SAncestralSampler, DPMPP2MSampler and LinearMultistepSampler keep
the reference's loops, evaluation order and random draws (one `noise_sampler(x)` per ancestral step, after the
step's evaluations, also on the last step).  On CUDA fp32 tensors with VanillaCFG or IdentityGuider the tail of
every denoiser evaluation -- the CFG combine, to_d, the step's update and any history term -- is one
ln3_sampler_step launch; the reference's per-sample `torch.where` selections become per-sample coefficients.
Otherwise the reference's torch arithmetic runs in the reference's op order.
"""
import torch

from .... import ops
from ...util import append_dims, default, instantiate_from_config
from .guiders import IdentityGuider, VanillaCFG
from .sampling_utils import get_ancestral_step, linear_multistep_coeff, to_d, to_neg_log_sigma, to_sigma

DEFAULT_GUIDER = {"target": "sgm.modules.diffusionmodules.guiders.IdentityGuider"}


class BaseDiffusionSampler:
    def __init__(self, discretization_config, num_steps=None, guider_config=None, verbose=False,
                 device="cuda"):
        self.num_steps = num_steps
        self.discretization = instantiate_from_config(discretization_config)
        self.guider = instantiate_from_config(default(guider_config, DEFAULT_GUIDER))
        self.verbose = verbose
        self.device = device

    def prepare_sampling_loop(self, x, cond, uc=None, num_steps=None):
        sigmas = self.discretization(self.num_steps if num_steps is None else num_steps, device=self.device)
        uc = default(uc, cond)
        x *= torch.sqrt(1.0 + sigmas[0] ** 2.0)
        num_sigmas = len(sigmas)
        s_in = x.new_ones([x.shape[0]])
        return x, s_in, sigmas, num_sigmas, cond, uc

    def denoise(self, x, denoiser, sigma, cond, uc):
        denoised = denoiser(*self.guider.prepare_inputs(x, sigma, cond, uc))
        return self.guider(denoised, sigma)

    def get_sigma_gen(self, num_sigmas):
        return range(num_sigmas - 1)

    # ---- fused tail (ln3_sampler_step) shared by the samplers below
    def _fusable(self, x):
        return x.is_cuda and x.dtype == torch.float32 and isinstance(self.guider, (VanillaCFG, IdentityGuider))

    def _denoise_halves(self, x, denoiser, sigma, cond, uc):
        """The denoiser output before the guider: (D_u, D_c or None, w_u, w_c) with guided D = w_u D_u + w_c D_c."""
        den = denoiser(*self.guider.prepare_inputs(x, sigma, cond, uc)).float().contiguous()
        if isinstance(self.guider, VanillaCFG):
            d_u, d_c = den.chunk(2)
            return d_u, d_c, 1.0 - self.guider.scale, self.guider.scale
        return den, None, 1.0, 0.0

    @staticmethod
    def _coef(x, k0=0.0, k1=0.0, k2=0.0, a=0.0, b=0.0, c=0.0, h0=0.0, h1=0.0, h2=0.0, s=0.0):
        """(B, 12) coefficient rows of ln3_sampler_step from per-sample tensors or scalars."""
        B = x.shape[0]
        col = lambda v: torch.broadcast_to(torch.as_tensor(v, device=x.device).float(), (B,))
        return torch.stack([col(v) for v in (k0, k1, k2, a, b, c, h0, h1, h2, s, 0.0, 0.0)], 1).contiguous()

    @staticmethod
    def _step(x, x_eval, coef, halves, hist=(), noise=None, x_out=True, hist_out=False):
        """One ln3_sampler_step on the guided denoiser halves; returns (x_out, hist_out) (new tensors or None)."""
        d_u, d_c = halves[0], halves[1]
        xo = torch.empty_like(x_eval) if x_out else None
        ho = torch.empty_like(x_eval) if hist_out else None
        ops.sampler_step(x.contiguous(), x_eval.contiguous(), coef, d_u, d_c, hist, noise, x_out=xo, hist_out=ho)
        return xo, ho


class SingleStepDiffusionSampler(BaseDiffusionSampler):
    def euler_step(self, x, d, dt):
        return x + dt * d


class EDMSampler(SingleStepDiffusionSampler):
    def __init__(self, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.s_churn, self.s_tmin, self.s_tmax, self.s_noise = s_churn, s_tmin, s_tmax, s_noise

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, gamma=0.0):
        sigma_hat = sigma * (gamma + 1.0)
        if gamma > 0:
            eps = torch.randn_like(x) * self.s_noise
            x = x + eps * append_dims(sigma_hat ** 2 - sigma ** 2, x.ndim) ** 0.5
        if x.is_cuda and x.dtype == torch.float32 and isinstance(self.guider, (VanillaCFG, IdentityGuider)):
            den = denoiser(*self.guider.prepare_inputs(x, sigma_hat, cond, uc)).float().contiguous()
            r = (next_sigma - sigma_hat) / sigma_hat          # dt / sigma, per sample
            if isinstance(self.guider, VanillaCFG):
                g = self.guider.scale
                d_u, d_c = den.chunk(2)
                coef = torch.stack([1 + r, -r * (1 - g), -r * g, torch.zeros_like(r)], 1)
                x_next = ops.sampler_affine_update(x.contiguous(), coef.float().contiguous(), d_u, d_c)
            else:
                coef = torch.stack([1 + r, -r, torch.zeros_like(r), torch.zeros_like(r)], 1)
                x_next = ops.sampler_affine_update(x.contiguous(), coef.float().contiguous(), den)
            return self.possible_correction_step(x_next, x, None, None, next_sigma, denoiser, cond, uc)
        denoised = self.denoise(x, denoiser, sigma_hat, cond, uc)
        d = to_d(x, sigma_hat, denoised)
        dt = append_dims(next_sigma - sigma_hat, x.ndim)
        euler_step = self.euler_step(x, d, dt)
        return self.possible_correction_step(euler_step, x, d, dt, next_sigma, denoiser, cond, uc)

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        for i in self.get_sigma_gen(num_sigmas):
            gamma = (min(self.s_churn / (num_sigmas - 1), 2 ** 0.5 - 1)
                     if self.s_tmin <= sigmas[i] <= self.s_tmax else 0.0)
            x = self.sampler_step(s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, uc, gamma)
        return x


class EulerEDMSampler(EDMSampler):
    def possible_correction_step(self, euler_step, x, d, dt, next_sigma, denoiser, cond, uc):
        return euler_step


class HeunEDMSampler(EDMSampler):
    def possible_correction_step(self, euler_step, x, d, dt, next_sigma, denoiser, cond, uc):
        if torch.sum(next_sigma) < 1e-14:
            return euler_step
        denoised = self.denoise(euler_step, denoiser, next_sigma, cond, uc)
        d_new = to_d(euler_step, next_sigma, denoised)
        d_prime = (d + d_new) / 2.0
        return torch.where(append_dims(next_sigma, x.ndim) > 0.0, x + d_prime * dt, euler_step)

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, gamma=0.0):
        if not self._fusable(x):
            return EDMSampler.sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc, gamma)
        sigma_hat = sigma * (gamma + 1.0)
        if gamma > 0:
            eps = torch.randn_like(x) * self.s_noise
            x = x + eps * append_dims(sigma_hat ** 2 - sigma ** 2, x.ndim) ** 0.5
        hv = self._denoise_halves(x, denoiser, sigma_hat, cond, uc)
        dt = next_sigma - sigma_hat
        # predictor: x_euler = x + dt d, d = (x - D) / sigma_hat kept for the corrector
        pred = self._coef(x, 1 / sigma_hat, -hv[2] / sigma_hat, -hv[3] / sigma_hat, a=1.0, c=dt)
        if torch.sum(next_sigma) < 1e-14:
            return self._step(x, x, pred, hv)[0]
        x_euler, d = self._step(x, x, pred, hv, hist_out=True)
        hv2 = self._denoise_halves(x_euler, denoiser, next_sigma, cond, uc)
        # corrector: x + (d + d_new)/2 dt where next_sigma > 0, else x_euler (sampling.py:231-233)
        on = next_sigma > 0.0
        sn = torch.where(on, next_sigma, torch.ones_like(next_sigma))
        z = torch.zeros_like(next_sigma)
        half_dt = torch.where(on, dt / 2.0, z)
        corr = self._coef(x, torch.where(on, 1 / sn, z), torch.where(on, -hv2[2] / sn, z),
                          torch.where(on, -hv2[3] / sn, z), a=on.float(), b=(~on).float(), c=half_dt, h0=half_dt)
        return self._step(x, x_euler, corr, hv2, hist=(d,))[0]


class AncestralSampler(SingleStepDiffusionSampler):
    def __init__(self, eta=1.0, s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.eta = eta
        self.s_noise = s_noise
        self.noise_sampler = lambda x: torch.randn_like(x)

    def ancestral_euler_step(self, x, denoised, sigma, sigma_down):
        d = to_d(x, sigma, denoised)
        dt = append_dims(sigma_down - sigma, x.ndim)
        return self.euler_step(x, d, dt)

    def ancestral_step(self, x, sigma, next_sigma, sigma_up):
        return torch.where(append_dims(next_sigma, x.ndim) > 0.0,
                           x + self.noise_sampler(x) * self.s_noise * append_dims(sigma_up, x.ndim), x)

    def _noise_scale(self, next_sigma, sigma_up):
        """The fused noise weight: s_noise * sigma_up where next_sigma > 0 (ancestral_step's torch.where)."""
        up = torch.as_tensor(sigma_up, device=next_sigma.device).float()
        return torch.where(next_sigma > 0.0, self.s_noise * up, torch.zeros_like(next_sigma))

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        for i in self.get_sigma_gen(num_sigmas):
            x = self.sampler_step(s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, uc)
        return x


class EulerAncestralSampler(AncestralSampler):
    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc):
        sigma_down, sigma_up = get_ancestral_step(sigma, next_sigma, eta=self.eta)
        if self._fusable(x):
            hv = self._denoise_halves(x, denoiser, sigma, cond, uc)
            noise = self.noise_sampler(x)
            r = (sigma_down - sigma) / sigma
            coef = self._coef(x, 0.0, hv[2], hv[3], a=1 + r, c=-r, s=self._noise_scale(next_sigma, sigma_up))
            return self._step(x, x, coef, hv, noise=noise.float().contiguous())[0]
        denoised = self.denoise(x, denoiser, sigma, cond, uc)
        x = self.ancestral_euler_step(x, denoised, sigma, sigma_down)
        return self.ancestral_step(x, sigma, next_sigma, sigma_up)


class DPMPP2SAncestralSampler(AncestralSampler):
    def get_variables(self, sigma, sigma_down):
        t, t_next = [to_neg_log_sigma(s) for s in (sigma, sigma_down)]
        h = t_next - t
        s = t + 0.5 * h
        return h, s, t, t_next

    def get_mult(self, h, s, t, t_next):
        mult1 = to_sigma(s) / to_sigma(t)
        mult2 = (-0.5 * h).expm1()
        mult3 = to_sigma(t_next) / to_sigma(t)
        mult4 = (-h).expm1()
        return mult1, mult2, mult3, mult4

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, **kwargs):
        sigma_down, sigma_up = get_ancestral_step(sigma, next_sigma, eta=self.eta)
        if self._fusable(x):
            return self._fused_step(sigma, next_sigma, sigma_down, sigma_up, denoiser, x, cond, uc)
        denoised = self.denoise(x, denoiser, sigma, cond, uc)
        x_euler = self.ancestral_euler_step(x, denoised, sigma, sigma_down)
        if torch.sum(sigma_down) < 1e-14:
            x = x_euler
        else:
            h, s, t, t_next = self.get_variables(sigma, sigma_down)
            mult = [append_dims(mult, x.ndim) for mult in self.get_mult(h, s, t, t_next)]
            x2 = mult[0] * x - mult[1] * denoised
            denoised2 = self.denoise(x2, denoiser, to_sigma(s), cond, uc)
            x_dpmpp2s = mult[2] * x - mult[3] * denoised2
            x = torch.where(append_dims(sigma_down, x.ndim) > 0.0, x_dpmpp2s, x_euler)
        return self.ancestral_step(x, sigma, next_sigma, sigma_up)

    def _fused_step(self, sigma, next_sigma, sigma_down, sigma_up, denoiser, x, cond, uc):
        hv = self._denoise_halves(x, denoiser, sigma, cond, uc)
        r = (sigma_down - sigma) / sigma                       # x_euler = (1 + r) x - r D
        if torch.sum(sigma_down) < 1e-14:
            noise = self.noise_sampler(x)
            coef = self._coef(x, 0.0, hv[2], hv[3], a=1 + r, c=-r, s=self._noise_scale(next_sigma, sigma_up))
            return self._step(x, x, coef, hv, noise=noise.float().contiguous())[0]
        h, s, t, t_next = self.get_variables(sigma, sigma_down)
        m1, m2, m3, m4 = self.get_mult(h, s, t, t_next)
        # x2 = mult1 x - mult2 D; D is kept for the samples whose sigma_down is 0 (they take x_euler)
        x2, den = self._step(x, x, self._coef(x, 0.0, hv[2], hv[3], a=m1, c=-m2), hv, hist_out=True)
        hv2 = self._denoise_halves(x2, denoiser, to_sigma(s), cond, uc)
        noise = self.noise_sampler(x)
        on = sigma_down > 0.0
        z = torch.zeros_like(sigma)
        coef = self._coef(x, 0.0, hv2[2], hv2[3], a=torch.where(on, m3, 1 + r), c=torch.where(on, -m4, z),
                          h0=torch.where(on, z, -r), s=self._noise_scale(next_sigma, sigma_up))
        return self._step(x, x2, coef, hv2, hist=(den,), noise=noise.float().contiguous())[0]


class DPMPP2MSampler(BaseDiffusionSampler):
    def get_variables(self, sigma, next_sigma, previous_sigma=None):
        t, t_next = [to_neg_log_sigma(s) for s in (sigma, next_sigma)]
        h = t_next - t
        if previous_sigma is not None:
            h_last = t - to_neg_log_sigma(previous_sigma)
            r = h_last / h
            return h, r, t, t_next
        return h, None, t, t_next

    def get_mult(self, h, r, t, t_next, previous_sigma):
        mult1 = to_sigma(t_next) / to_sigma(t)
        mult2 = (-h).expm1()
        if previous_sigma is not None:
            mult3 = 1 + 1 / (2 * r)
            mult4 = 1 / (2 * r)
            return mult1, mult2, mult3, mult4
        return mult1, mult2

    def sampler_step(self, old_denoised, previous_sigma, sigma, next_sigma, denoiser, x, cond, uc=None):
        if self._fusable(x):
            return self._fused_step(old_denoised, previous_sigma, sigma, next_sigma, denoiser, x, cond, uc)
        denoised = self.denoise(x, denoiser, sigma, cond, uc)
        h, r, t, t_next = self.get_variables(sigma, next_sigma, previous_sigma)
        mult = [append_dims(mult, x.ndim) for mult in self.get_mult(h, r, t, t_next, previous_sigma)]
        x_standard = mult[0] * x - mult[1] * denoised
        if old_denoised is None or torch.sum(next_sigma) < 1e-14:
            return x_standard, denoised
        denoised_d = mult[2] * denoised - mult[3] * old_denoised
        x_advanced = mult[0] * x - mult[1] * denoised_d
        x = torch.where(append_dims(next_sigma, x.ndim) > 0.0, x_advanced, x_standard)
        return x, denoised

    def _fused_step(self, old_denoised, previous_sigma, sigma, next_sigma, denoiser, x, cond, uc):
        hv = self._denoise_halves(x, denoiser, sigma, cond, uc)
        h, r, t, t_next = self.get_variables(sigma, next_sigma, previous_sigma)
        mult = self.get_mult(h, r, t, t_next, previous_sigma)
        if old_denoised is None or torch.sum(next_sigma) < 1e-14:
            coef = self._coef(x, 0.0, hv[2], hv[3], a=mult[0], c=-mult[1])
            return self._step(x, x, coef, hv, hist_out=True)
        # x_advanced = mult1 x - mult2 (mult3 D - mult4 D_old) where next_sigma > 0, else x_standard
        on = next_sigma > 0.0
        z = torch.zeros_like(sigma)
        coef = self._coef(x, 0.0, hv[2], hv[3], a=mult[0], c=torch.where(on, -mult[1] * mult[2], -mult[1]),
                          h0=torch.where(on, mult[1] * mult[3], z))
        return self._step(x, x, coef, hv, hist=(old_denoised.float().contiguous(),), hist_out=True)

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        old_denoised = None
        for i in self.get_sigma_gen(num_sigmas):
            x, old_denoised = self.sampler_step(old_denoised, None if i == 0 else s_in * sigmas[i - 1],
                                                s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, uc=uc)
        return x


class LinearMultistepSampler(BaseDiffusionSampler):
    def __init__(self, order=4, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.order = order

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        ds = []
        sigmas_cpu = sigmas.detach().cpu().numpy()
        fused = self._fusable(x) and not kwargs and self.order <= 4
        for i in self.get_sigma_gen(num_sigmas):
            sigma = s_in * sigmas[i]
            cur_order = min(i + 1, self.order)
            coeffs = [linear_multistep_coeff(cur_order, sigmas_cpu, i, j) for j in range(cur_order)]
            if fused:
                # d = (x - D) / sigma into the history, x + sum_j coeff_j d_{i-j} in the same launch
                hv = self._denoise_halves(x, denoiser, sigma, cond, uc)
                past = list(reversed(ds))[:cur_order - 1]
                coef = self._coef(x, 1 / sigma, -hv[2] / sigma, -hv[3] / sigma, a=1.0, c=coeffs[0],
                                  **{f"h{j}": coeffs[j + 1] for j in range(cur_order - 1)})
                x, d = self._step(x, x, coef, hv, hist=past, hist_out=True)
                ds.append(d)
                if len(ds) > self.order:
                    ds.pop(0)
                continue
            denoised = denoiser(*self.guider.prepare_inputs(x, sigma, cond, uc), **kwargs)
            denoised = self.guider(denoised, sigma)
            d = to_d(x, sigma, denoised)
            ds.append(d)
            if len(ds) > self.order:
                ds.pop(0)
            x = x + sum(coeff * d for coeff, d in zip(coeffs, reversed(ds)))
        return x

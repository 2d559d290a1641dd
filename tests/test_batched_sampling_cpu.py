"""CPU tests of batched `sample()` argument handling: prompt / guidance / zT normalisation and its errors, the per-row
guidance mix of the op-by-op loops, the per-row SDXL added conditioning, per-image latent draws, and the batching and
zT order of examples/text_to_mscoco.py. No GPU compute here."""
import pytest
import torch

from cfgpp_b200 import batching as Bt
from cfgpp_b200 import kdiffusion as K
from cfgpp_b200 import schedule as S
from cfgpp_b200.conditioning import SyntheticTextEncoder
from oracle import samplers as OSm, schedule as OS


def test_normalize_batch_shapes_and_broadcast():
    B, p, g = Bt.normalize_batch({"null": "", "text": "a cat"}, 7.5)
    assert (B, p, g) == (1, {"null": "", "text": "a cat"}, 7.5)
    B, p, g = Bt.normalize_batch({"null": "", "text": ["a", "b", "c"]}, 0.6)
    assert B == 3 and p == {"null": "", "text": ["a", "b", "c"]} and g == 0.6
    B, p, g = Bt.normalize_batch({"null": ["x", "y"], "text": ("a", "b")}, [0.0, 1.0], torch.zeros(2, 4, 8, 8))
    assert B == 2 and p["text"] == ["a", "b"] and g == [0.0, 1.0]
    # a lambda sweep over one prompt: the strings are broadcast
    B, p, g = Bt.normalize_batch({"null": "", "text": "a cat"}, (0.2, 0.4, 0.6, 0.8))
    assert B == 4 and p["text"] == "a cat" and g == [0.2, 0.4, 0.6, 0.8]
    # equal entries are the scalar call
    assert Bt.normalize_batch({"text": ["a", "b"]}, [0.6, 0.6])[2] == 0.6
    assert Bt.normalize_batch({"text": "a"}, [0.6])[2] == 0.6
    # zT alone sets the batch
    assert Bt.normalize_batch({"text": "a"}, 0.6, torch.zeros(3, 4, 8, 8))[0] == 3


@pytest.mark.parametrize("prompts,guidance,zT,match", [
    ({"null": ["x", "y", "z"], "text": ["a", "b"]}, 0.6, None, "batch sizes differ"),
    ({"null": "", "text": ["a", "b"]}, [0.1, 0.2, 0.3], None, "cfg_guidance=3"),
    ({"null": "", "text": ["a", "b"]}, 0.6, torch.zeros(3, 4, 8, 8), "zT=3"),
    ({"null": "", "text": "a"}, [0.1, 0.2], torch.zeros(1, 4, 8, 8), "batch sizes differ"),
    ({"null": "", "text": []}, 0.6, None, "empty batch"),
    ({"null": "", "text": ["a", 3]}, 0.6, None, "list of strings"),
    ({"null": "", "text": "a"}, 0.6, torch.zeros(4, 8, 8), "zT must be"),
])
def test_normalize_batch_rejects_mismatches(prompts, guidance, zT, match):
    with pytest.raises(ValueError, match=match):
        Bt.normalize_batch(prompts, guidance, zT)


def test_guidance_helpers_and_step_table_scalar():
    assert Bt.guidance_table(0.6) is None and Bt.guidance_table((0.0, 1.0)) == [0.0, 1.0]
    assert Bt.guidance_values(7.5) == [7.5] and Bt.schedule_lambda([0.3, 0.9]) == 0.3
    sch = S.Schedule.make(10)
    scalar = S.ddim_cfgpp_steps(sch, 0.3, True)
    table = S.ddim_cfgpp_steps(sch, [0.3, 0.9], True)
    assert all(bytes(a) == bytes(b) for a, b in zip(scalar, table))


def test_guidance_mix_rows_round_as_their_scalar_calls():
    g = torch.Generator().manual_seed(0)
    eu = torch.randn(3, 4, 8, 8, generator=g).half()
    ec = torch.randn(3, 4, 8, 8, generator=g).half()
    lams = [0.0, 0.6, 7.5]
    mixed = Bt.guidance_mix(eu, ec, lams)
    for b, lam in enumerate(lams):
        assert torch.equal(mixed[b:b + 1], eu[b:b + 1] + lam * (ec[b:b + 1] - eu[b:b + 1]))
    assert torch.equal(Bt.guidance_mix(eu, ec, 0.6), eu + 0.6 * (ec - eu))
    with pytest.raises(ValueError):
        Bt.guidance_mix(eu, ec, [0.1, 0.2])


class _FakeUNet:
    """Row-independent stand-in with the diffusers call signature (as in test_kdiffusion_cpu)."""
    def __call__(self, z, t, encoder_hidden_states=None, added_cond_kwargs=None):
        t = t.reshape(-1, 1, 1, 1).to(z.dtype)
        ctx = encoder_hidden_states.float().mean(dim=(1, 2)).reshape(-1, 1, 1, 1).to(z.dtype)
        return {"sample": torch.tanh(z * (0.5 + t / 1000)) * 0.8 + 0.3 * ctx}


class _StubSolver(K.KDiffusionMixin):
    def __init__(self, tb):
        self.log_sigmas, self.total_alphas, self.device = tb.log_sigmas, tb.total_alphas, torch.device("cpu")
        self.unet, self.decode = _FakeUNet(), None

    def predict_noise(self, zt, t, uc, c, added_cond_kwargs=None):
        tt = t.reshape(1).expand(zt.shape[0])
        return self.unet(zt, tt, uc)["sample"], self.unet(zt, tt, c)["sample"]


@pytest.mark.parametrize("loop", ["euler", "dpmpp_2m"])
def test_op_by_op_loop_with_per_image_guidance_equals_row_runs(loop):
    """The op-by-op k-diffusion loops apply a per-image lambda row by row: row b of a batch is bit-identical to the
    same loop run on row b alone with the scalar lambda[b]."""
    tb = OS.make_tables(6)
    g = torch.Generator().manual_seed(3)
    noise = torch.randn(3, 4, 8, 8, generator=g)
    uc = torch.randn(3, 77, 16, generator=g).half()
    c = torch.randn(3, 77, 16, generator=g).half()
    sigmas = OSm.karras_sigmas(tb)
    x0 = OSm.kd_start_state(noise, sigmas)
    fn = {"euler": K.euler_cfgpp_loop, "dpmpp_2m": K.dpmpp_2m_cfgpp_karras_loop}[loop]
    lams = [0.0, 0.6, 1.0]
    s = _StubSolver(tb)
    d, x = fn(s, x0.clone(), sigmas, lams, (uc, c))
    for b, lam in enumerate(lams):
        db, xb = fn(s, x0[b:b + 1].clone(), sigmas, lam, (uc[b:b + 1], c[b:b + 1]))
        assert torch.equal(x[b:b + 1], xb) and torch.equal(d[b:b + 1], db), f"row {b}"


def test_sdxl_added_conditions_per_row():
    P = 4
    neg_p = torch.arange(3 * P, dtype=torch.float16).reshape(3, P) * -1 - 1
    pos_p = torch.arange(3 * P, dtype=torch.float16).reshape(3, P) + 1
    neg_t = torch.tensor([[512, 512, 0, 0, 512, 512]], dtype=torch.float16)
    pos_t = torch.tensor([[1024, 1024, 0, 0, 1024, 1024]], dtype=torch.float16)
    # scalar, one image: the reference's tensors (latent_sdxl.py:249-257)
    te, ti = Bt.sdxl_added_conditions(neg_p[:1], pos_p[:1], neg_t, pos_t, 0.6, 1)
    assert torch.equal(te, torch.cat([neg_p[:1], pos_p[:1]])) and torch.equal(ti, torch.cat([neg_t, pos_t]))
    for lam in (0.0, 1.0):
        te, ti = Bt.sdxl_added_conditions(neg_p[:1], pos_p[:1], neg_t, pos_t, lam, 1)
        assert torch.equal(te, pos_p[:1]) and torch.equal(ti, pos_t)
    # scalar, a batch: one time-id row per image
    te, ti = Bt.sdxl_added_conditions(neg_p, pos_p, neg_t, pos_t, 0.6, 3)
    assert torch.equal(te, torch.cat([neg_p, pos_p])) and torch.equal(ti, torch.cat([neg_t.expand(3, -1),
                                                                                        pos_t.expand(3, -1)]))
    te, ti = Bt.sdxl_added_conditions(neg_p, pos_p, neg_t, pos_t, 1.0, 3)
    assert te.shape == (3, P) and torch.equal(ti, pos_t.expand(3, -1))
    # per image: lambda in {0, 1} -> the uncond row takes the positive embedding, otherwise the negative one
    te, ti = Bt.sdxl_added_conditions(neg_p, pos_p, neg_t, pos_t, [0.0, 0.6, 1.0], 3)
    assert te.shape == (6, P) and ti.shape == (6, 6)
    assert torch.equal(te[:3], torch.stack([pos_p[0], neg_p[1], pos_p[2]])) and torch.equal(te[3:], pos_p)
    assert torch.equal(ti[:3], torch.cat([pos_t, neg_t, pos_t])) and torch.equal(ti[3:], pos_t.expand(3, -1))
    # each image's rows are those of its own single-image call
    for b, lam in enumerate([0.0, 0.6, 1.0]):
        te1, ti1 = Bt.sdxl_added_conditions(neg_p[b:b + 1], pos_p[b:b + 1], neg_t, pos_t, lam, 1)
        assert torch.equal(te1[0], te[b]) and torch.equal(te1[-1], te[3 + b])
        assert torch.equal(ti1[0], ti[b]) and torch.equal(ti1[-1], ti[3 + b])


def test_latents_are_drawn_one_image_at_a_time():
    torch.manual_seed(5)
    batch = Bt.draw_latents((3, 4, 8, 8))
    torch.manual_seed(5)
    serial = [torch.randn(1, 4, 8, 8) for _ in range(3)]
    assert torch.equal(batch, torch.cat(serial))
    torch.manual_seed(5)
    assert torch.equal(Bt.draw_latents((1, 4, 8, 8)), serial[0])


def test_prompt_lists_encode_one_row_per_prompt():
    from cfgpp_b200 import latent_diffusion as LD, latent_sdxl as LX
    sd = object.__new__(LD.BaseDDIMCFGpp)
    sd.text_encoder, sd.device = SyntheticTextEncoder(16), torch.device("cpu")
    uc, c, g, zT = sd.batch_inputs(["", ["a", "b", "c"]], [0.0, 0.6, 1.0])
    assert uc.shape == c.shape == (3, 77, 16) and g == [0.0, 0.6, 1.0] and zT is None
    for b, p in enumerate("abc"):
        assert torch.equal(c[b:b + 1], sd.text_encoder(p, "cpu")[0])
        assert torch.equal(uc[b:b + 1], sd.text_encoder("", "cpu")[0])
    with pytest.raises(ValueError, match="batch sizes differ"):
        sd.sample(prompt=[["", ""], ["a", "b", "c"]], cfg_guidance=0.6)
    xl = object.__new__(LX.BaseDDIMCFGpp)
    xl.text_enc_1, xl.text_enc_2 = SyntheticTextEncoder(8, 0), SyntheticTextEncoder(8, 12)
    xl.device = torch.device("cpu")
    nu, pe, pn, pp = xl.get_text_embed("", ["a", "b"], "", ["a", "b"], batch=2)
    assert nu.shape == pe.shape == (2, 77, 16) and pn.shape == pp.shape == (2, 12)
    assert torch.equal(pp[1:], xl.text_enc_2("b", "cpu")[1]) and torch.equal(pn[1:], xl.text_enc_2("", "cpu")[1])
    xl.default_sample_size, xl.vae_scale_factor = 8, 8
    with pytest.raises(ValueError, match="batch sizes differ"):
        xl.sample(prompt1=["", ["a", "b"]], prompt2=["", ["a", "b", "c"]], cfg_guidance=0.6)


@pytest.mark.parametrize("world", [1, 3])
def test_mscoco_batches_keep_each_image_zT(world):
    from examples.text_to_mscoco import rank_batches
    n, latent = 11, (1, 4, 4, 4)
    torch.manual_seed(42)
    ref = [torch.randn(latent) for _ in range(n)]
    for bs in (1, 2, 4, 8):
        seen = {}
        for rank in range(world):
            torch.manual_seed(42)
            for idx, zT in rank_batches(n, rank, world, bs, latent):
                assert 1 <= len(idx) <= bs and zT.shape == (len(idx), *latent[1:])
                assert all(i % world == rank for i in idx) and idx == sorted(idx)
                for j, i in enumerate(idx):
                    seen[i] = zT[j:j + 1]
        assert sorted(seen) == list(range(n))
        assert all(torch.equal(seen[i], ref[i]) for i in range(n)), f"batch_size={bs} world={world}"
    with pytest.raises(ValueError):
        next(rank_batches(n, 0, 1, 0, latent))


def test_lightning_guidance_assertion_checks_every_entry():
    from cfgpp_b200 import latent_sdxl as LX
    lt = object.__new__(LX.BaseDDIMCFGppLight)
    with pytest.raises(AssertionError, match="CFG should be turned off"):
        lt.reverse_process(None, None, [1.0, 0.6], None)

"""`ldm.models.diffusion.plms.PLMSSampler` import target (scripts/stable_txt2img.py:19 imports it unconditionally).
The PLMS sampler is not on the CelebBasis hot path (SURVEY.md section 2: the reference's test scripts run DDIM,
02_start_test.sh:36-41), so only the name exists here."""


class PLMSSampler:
    def __init__(self, model, schedule="linear", **kwargs):
        raise NotImplementedError("PLMSSampler is out of scope for the H100 path: use DDIMSampler (--plms off)")

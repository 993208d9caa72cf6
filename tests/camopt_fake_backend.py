"""TEST SCAFFOLDING ONLY -- tests/fake_backend.py's CPU stand-in for B200Backend, plus the two camera-pose gradient
leaves (neurad_encoding_mean_bwd, isotropic_gaussian_bwd) backed by the host emulation of their device code
(tests/camopt_emul.py)."""
from oracle import neurad_oracle as O
from tests import camopt_emul
from tests.fake_backend import FakeBackend


class CamoptFakeBackend(FakeBackend):
    def neurad_encoding_mean_bwd(self, field, mean, std, times, dfeatures=None, density=None, ddensity=None, flip=None):
        return camopt_emul.encoding_mean_bwd(self.cfg, self.params, O.pdf_u, field, mean, std, times, dfeatures, density, ddensity, flip)

    def isotropic_gaussian_bwd(self, bins_e, dmean):
        return camopt_emul.gaussian_bwd(bins_e, dmean)

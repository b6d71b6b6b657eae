from .cglb import CGLB
from .gplvm import BayesianGPLVM
from .gpr import GPR
from .model import BayesianModel, GPModel
from .sgpr import GPRFITC, SGPR
from .svgp import SVGP
from .vgp import VGP, VGPOpperArchambeau


def maximum_log_likelihood_objective(model, data=None):
    return model.maximum_log_likelihood_objective() if data is None else model.maximum_log_likelihood_objective(data)


def training_loss_closure(model, data=None, **kw):
    return model.training_loss_closure(**kw) if data is None else model.training_loss_closure(data, **kw)


__all__ = ["BayesianGPLVM", "BayesianModel", "CGLB", "GPModel", "GPR", "GPRFITC", "SGPR", "SVGP", "VGP", "VGPOpperArchambeau",
           "maximum_log_likelihood_objective",
           "training_loss_closure"]

"""stochvolmodels_b200 -- H100-native (sm_90a CUDA) engine for the two numerical hot paths of ArturSepp/StochVolModels,
behind the reference's Pricer API.  See DESIGN.md / INTEGRATION.md.  There is no CPU fallback: computing needs
``lib/libb200sv.so`` (built by ``python -m stochvolmodels_b200._build``) and a CUDA device."""
from .data.option_chain import OptionChain, OptionSlice, get_btc_test_chain_data
from .engine import HAWKES_GREEK_PARAMS, HAWKES_RISK_PREMIA_GREEK_PARAMS, infer_bsm_ivols_from_model_chain_prices, infer_bsm_ivols_from_slice_prices
from .pricers.calibration import CalibrationEngine, CalibrationError, ConstraintsType, LogsvModelCalibrationType
from .pricers.hawkes_jd_pricer import HawkesJDParams, HawkesJDPricer
from .pricers.fourier_greeks import ChainIvolGreeks, ChainIvolHessian, FourierChainGreeks, FourierChainHessian
from .pricers.heston_pricer import BTC_HESTON_PARAMS, HestonParams, HestonPricer
from .pricers.logsv.affine_expansion import ExpansionOrder
from .pricers.logsv.vol_moments import compute_analytic_qvar
from .pricers.logsv_pricer import LOGSV_BTC_PARAMS, LogSvParams, LogSVPricer
from .pricers.mc_greeks import McChainGreeks
from .pricers.model_pricer import ModelParams, ModelPricer
from .utils.config import OptionType, VariableType
from .utils.funcs import set_seed, set_time_grid
from .utils.mgf_pricer import compute_integration_weights

__version__ = "0.1.0"
__all__ = ["HawkesJDParams", "HawkesJDPricer", "OptionChain", "get_btc_test_chain_data", "HestonParams", "HestonPricer", "BTC_HESTON_PARAMS", "ExpansionOrder",
           "LogSvParams", "LogSVPricer", "CalibrationEngine", "CalibrationError", "ConstraintsType", "LogsvModelCalibrationType", "LOGSV_BTC_PARAMS", "ModelParams", "ModelPricer", "OptionType", "VariableType", "set_seed", "set_time_grid",
           "compute_integration_weights", "OptionSlice", "compute_analytic_qvar", "infer_bsm_ivols_from_slice_prices",
           "infer_bsm_ivols_from_model_chain_prices", "McChainGreeks", "FourierChainGreeks", "FourierChainHessian",
           "ChainIvolGreeks", "ChainIvolHessian", "HAWKES_GREEK_PARAMS", "HAWKES_RISK_PREMIA_GREEK_PARAMS"]

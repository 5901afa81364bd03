"""ModelPricer: the plugin boundary of the reference (pricers/model_pricer.py:83-265), same method names, argument meaning,
defaults and return shapes.  Concrete pricers implement ``price_chain`` / ``model_mc_price_chain`` / ``simulate_terminal_values``
on top of libb200sv; everything else here is inherited host logic.  Plotting methods (:279-631) are presentation and out of
scope (SURVEY.md §2 row 6)."""
from __future__ import annotations

from abc import ABC, abstractmethod
from dataclasses import asdict, dataclass
from typing import List, Tuple

import numpy as np

from ..data.option_chain import OptionChain
from ..utils.config import VariableType


@dataclass
class ModelParams:
    """abstract parameter container (reference pricers/model_pricer.py:29-42)."""

    @classmethod
    def copy(cls, obj: "ModelParams") -> "ModelParams":
        return cls(**asdict(obj))


class ModelPricer(ABC):
    def __init__(self):
        super().__init__()

    # ---- generic interfaces ---------------------------------------------------------------------------------------------
    @abstractmethod
    def price_chain(self, option_chain: OptionChain, params: ModelParams, **kwargs) -> List[np.ndarray]:
        """price a chain analytically (Fourier); one float64 array of prices per maturity."""

    def compute_chain_prices_with_vols(self, option_chain: OptionChain, params: ModelParams,
                                       variable_type: VariableType = VariableType.LOG_RETURN, **kwargs
                                       ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        """price chain and compute model vols (reference :109-120)."""
        model_prices = self.price_chain(option_chain=option_chain, params=params, variable_type=variable_type, **kwargs)
        model_ivols = option_chain.compute_model_ivols_from_chain_data(model_prices=model_prices)
        return model_prices, model_ivols

    def compute_chain_ivol_greeks(self, option_chain: OptionChain, params: ModelParams, with_theta: bool = False, **kwargs):
        """implied vols and their first-order sensitivities -> ``ChainIvolGreeks`` (DESIGN.md §4.6): ``self.price_chain_greeks`` with the
        same kwargs (and so its rejections, before any GPU work), then one GPU call that inverts the prices and maps the price rows to
        implied-vol rows.  The ivols are bit-identical to ``compute_chain_prices_with_vols`` with the same arguments; the rows are exact
        derivatives of them on the transform grid the pricer holds fixed.  ``with_theta``: also the ivol theta -d ivol / d ttm (§4.8), from
        ``price_chain_greeks(with_theta=True)`` and one more GPU call."""
        from .fourier_greeks import to_chain_ivol_sensitivities
        if with_theta:
            kwargs["with_theta"] = True
        return to_chain_ivol_sensitivities(option_chain, self.price_chain_greeks(option_chain, params, **kwargs))

    def compute_chain_ivol_hessian(self, option_chain: OptionChain, params: ModelParams, **kwargs):
        """``compute_chain_ivol_greeks`` plus the second order -> ``ChainIvolHessian``: from ``self.price_chain_hessian`` with the same
        kwargs (same ivols, bit for bit).  ``with_theta=True`` raises NotImplementedError, as ``price_chain_hessian`` does."""
        from .fourier_greeks import to_chain_ivol_sensitivities
        return to_chain_ivol_sensitivities(option_chain, self.price_chain_hessian(option_chain, params, **kwargs))

    def compute_model_ivols_for_chain(self, option_chain: OptionChain, params: ModelParams, **kwargs) -> List[np.ndarray]:
        _, model_ivols = self.compute_chain_prices_with_vols(option_chain=option_chain, params=params, **kwargs)
        return model_ivols

    def model_mc_price_chain(self, option_chain: OptionChain, params: ModelParams,
                             variable_type: VariableType = VariableType.LOG_RETURN, **kwargs
                             ) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        raise NotImplementedError("must be implemented in parent class")

    def calibrate_model_params_to_chain(self, option_chain: OptionChain, **kwargs):
        raise NotImplementedError("must be implemented in parent class")

    # ---- implemented on top of price_chain ---------------------------------------------------------------------------------
    def price_slice(self, params: ModelParams, ttm: float, forward: float, strikes: np.ndarray, optiontypes: np.ndarray,
                    discfactor: float = 1.0, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """price one slice through the chain pricer; returns (prices, implied vols) (reference :156-178)."""
        option_chain = OptionChain.slice_to_chain(ttm=ttm, forward=forward, strikes=strikes, optiontypes=optiontypes, discfactor=discfactor)
        model_prices = self.price_chain(option_chain=option_chain, params=params, **kwargs)
        model_ivols = option_chain.compute_model_ivols_from_chain_data(model_prices=model_prices)
        return model_prices[0], model_ivols[0]

    def price_vanilla(self, params: ModelParams, ttm: float, forward: float, strike: float, optiontype: str,
                      discfactor: float = 1.0, **kwargs) -> Tuple[float, float]:
        """price a single option; returns (price, implied vol) (reference :180-196)."""
        model_prices, model_ivols = self.price_slice(params=params, ttm=ttm, forward=forward, strikes=np.array([strike]),
                                                     optiontypes=np.array([optiontype]), discfactor=discfactor, **kwargs)
        return model_prices[0], model_ivols[0]

    # ---- monte carlo ------------------------------------------------------------------------------------------------------
    def simulate_vol_paths(self, params: ModelParams, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        raise NotImplementedError("must be implemented in parent class")

    def simulate_terminal_values(self, params: ModelParams, **kwargs) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        raise NotImplementedError("must be implemented in parent class")

    def compute_mc_chain_implied_vols(self, option_chain: OptionChain, params: ModelParams,
                                      variable_type: VariableType = VariableType.LOG_RETURN, nb_path: int = 100000, **kwargs):
        """MC prices with +-1.96 standard-error bands and their implied vols (reference :216-241)."""
        model_prices_ttms, option_std_ttms = self.model_mc_price_chain(option_chain=option_chain, params=params,
                                                                       variable_type=variable_type, nb_path=nb_path, **kwargs)
        std_factor = 1.96
        ups = [p + std_factor * s for p, s in zip(model_prices_ttms, option_std_ttms)]
        downs = [np.maximum(p - std_factor * s, 1e-10) for p, s in zip(model_prices_ttms, option_std_ttms)]
        ivols_mid = option_chain.compute_model_ivols_from_chain_data(model_prices=model_prices_ttms)
        ivols_up = option_chain.compute_model_ivols_from_chain_data(model_prices=ups)
        ivols_down = option_chain.compute_model_ivols_from_chain_data(model_prices=downs)
        return model_prices_ttms, ups, downs, ivols_mid, ivols_up, ivols_down, option_std_ttms

    # ---- densities ----------------------------------------------------------------------------------------------------------
    def get_log_return_mc_pdf(self, ttm: float, params: ModelParams, x_grid: np.ndarray, nb_path: int = 100000) -> np.ndarray:
        """normalised Gaussian-KDE histogram of simulated terminal log-returns on ``x_grid`` (reference :243-265): NaN and |value| > 1e16
        samples are counted, reported on stdout with the reference's wording and dropped.  Host post-processing of GPU samples.
        The reference hands the whole return value of ``simulate_terminal_values`` to the filter, which only works for pricers that
        return one array; a (log-return, vol, qvar) tuple -- what LogSVPricer / HestonPricer return -- is reduced to its log-returns."""
        from scipy import stats
        t_values = self.simulate_terminal_values(ttm=ttm, params=params, nb_path=nb_path)
        if isinstance(t_values, tuple):
            t_values = t_values[0]
        t_values = np.asarray(t_values, dtype=float)
        cut_off = 1e16
        nans = np.isnan(t_values)
        pos = ~nans & (t_values > cut_off)
        neg = ~nans & (t_values < -cut_off)
        print(f"in mc: num -inf = {np.sum(neg)}, num +inf = {np.sum(pos)}, num nans = {np.sum(nans)}")
        z = stats.gaussian_kde(t_values[~(nans | pos | neg)])(x_grid)
        return z / np.nansum(z)

    def compute_logreturn_pdf(self, params: ModelParams, **kwargs) -> np.ndarray:
        raise NotImplementedError("must be implemented in parent class")

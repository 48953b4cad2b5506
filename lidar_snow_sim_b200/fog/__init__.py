from .simulation import (ParameterSet, simulate_fog, simulate_fog_batch, load_integral_table,  # noqa: F401
                         get_available_alphas, integral_table, generate_integral_lookup_tables)
from .haze import BetaRadomization, haze_point_cloud  # noqa: F401

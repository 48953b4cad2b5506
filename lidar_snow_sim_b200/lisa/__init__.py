from .simulation import LISA, generate_mie_tables, mie_table  # noqa: F401

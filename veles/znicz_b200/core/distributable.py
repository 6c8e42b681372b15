"""IDistributable protocol (``veles.distributable``).

The reference's only parallelism is the 5-method master/slave contract
(/root/reference/nn_units.py:118,178-211,644-694). It is kept as API (tests drive
it in-process, and the multi-process CPU path can use it over gloo), while the
H100 data-parallel path is synchronous all-reduce fused with the update kernel
(``veles.znicz_b200.parallel``).
"""


class IDistributable(object):
    __required__ = ("generate_data_for_slave", "generate_data_for_master",
                    "apply_data_from_master", "apply_data_from_slave", "drop_slave")


class TriviallyDistributable(object):
    """Mixin: a unit with nothing to exchange."""

    def generate_data_for_slave(self, slave=None):
        return None

    def generate_data_for_master(self):
        return None

    def apply_data_from_master(self, data):
        pass

    def apply_data_from_slave(self, data, slave=None):
        pass

    def drop_slave(self, slave=None):
        pass

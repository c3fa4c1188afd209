"""multistate samplers on the GPU engine (mirrors openmmtools.multistate for the replica-exchange path)."""
from .multistatesampler import MultiStateSampler
from .replicaexchange import ReplicaExchangeSampler
from .paralleltempering import ParallelTemperingSampler
from .sams import SAMSSampler
from .utils import SimulationNaNError
from .multistatereporter import MultiStateReporter
from .multistateanalyzer import MultiStateSamplerAnalyzer, ReplicaExchangeAnalyzer, SAMSAnalyzer, MultiPhaseAnalyzer

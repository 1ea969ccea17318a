"""dada2_b200 -- H100-native (sm_90a CUDA) implementation of DADA2's dada() core loop behind the
reference's dada_uniques() interface.  See DESIGN.md / INTEGRATION.md."""
from . import api  # noqa: F401
from .api import Dada2bError, PackedCall, Resident, dada_uniques  # noqa: F401
from . import bimera  # noqa: F401,E402
from .bimera import isShiftDenovo, removeBimeraDenovo  # noqa: F401,E402
from . import merge  # noqa: F401,E402
from . import derep  # noqa: F401,E402
from . import errmodel  # noqa: F401,E402
from . import seqtab  # noqa: F401,E402
from . import filter  # noqa: F401,E402
from .filter import filterAndTrim, filter_reads  # noqa: F401,E402
from . import primer  # noqa: F401,E402
from .primer import removePrimers, remove_primers_reads  # noqa: F401,E402
from .errmodel import PacBioErrfun  # noqa: F401,E402
from .derep import pool_dereps  # noqa: F401,E402
from . import denoise  # noqa: F401,E402
from .denoise import dada, learnErrors  # noqa: F401,E402
from . import taxonomy  # noqa: F401,E402
from .taxonomy import TaxDB, assignTaxonomy  # noqa: F401,E402
from . import species  # noqa: F401,E402
from .species import SpeciesDB, addSpecies, assignSpecies  # noqa: F401,E402
from . import paired  # noqa: F401,E402
from .paired import mergePairs  # noqa: F401,E402
from . import align  # noqa: F401,E402
from .align import nwalign  # noqa: F401,E402
from . import qc  # noqa: F401,E402
from .qc import plotComplexity, plotQualityProfile  # noqa: F401,E402

from .views import load_image  # noqa: F401
from .gpu_views import GpuViewGenerator, sample_view_params  # noqa: F401,E402
from .paired import DistributedInfiniteSampler, FeatureStoreDataset, InMemoryPairs, InfiniteSampler  # noqa: F401,E402
from .resume import resumed_iter  # noqa: F401,E402

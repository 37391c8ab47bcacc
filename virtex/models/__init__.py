from virtex_b200.models import (CaptioningModel, ForwardCaptioningModel, BidirectionalCaptioningModel,  # noqa: F401
                                VirTexModel)
from virtex_b200.models import (ClassificationModel, TokenClassificationModel,  # noqa: F401
                                MultiLabelClassificationModel)

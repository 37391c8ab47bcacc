from virtex_b200.models import (ClassificationModel, TokenClassificationModel,  # noqa: F401
                                MultiLabelClassificationModel)

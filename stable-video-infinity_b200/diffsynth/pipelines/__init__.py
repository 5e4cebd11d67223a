from .svi_video import SVIVideoPipeline
from .wan_video import (WanRepalceAnyoneVideoPipeline, WanReplaceAnyoneVideoPipeline, WanUniAnimateLongVideoPipeline,
                        WanUniAnimateVideoPipeline, WanVideoPipeline)

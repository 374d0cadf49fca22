// REFERENCE denoiser (plain temporal accumulation of IN_SIGNAL into an RGBA32F history, copied to OUT_SIGNAL).
// Restates the reference's Source/Denoisers/Reference.hpp:11-90 (one permanent RGBA32F texture, two passes, the instance-wide
// accumulated-frame counter that restarts on any camera / rect / accumulation-mode change).
#include "scheduler.h"

#include <algorithm>
#include <cstring>

using namespace nrd;

namespace nrdb200
{
namespace
{
constexpr uint16_t R(ResourceType t) { return (uint16_t)t; }
enum ReferencePass : uint32_t { RF_ACCUMULATE = 0, RF_COPY = 1 };
} // namespace

void Scheduler::AddReference(DenoiserSlot& slot)
{
    new (&slot.settings.reference) ReferenceSettings();
    slot.settingsSize = sizeof(ReferenceSettings);
    const char* dn = "Reference";
    const uint16_t P_HISTORY = kPermanentBase;
    AddPermanent(Format::RGBA32_SFLOAT);

    BeginPass(dn, "Temporal accumulation");
    In(R(ResourceType::IN_SIGNAL));
    Out(P_HISTORY);
    Emit({Family::REFERENCE, Pass::TemporalAccumulation}, 16, 16, sizeof(ReferenceAccumulateConstants));

    BeginPass(dn, "Copy");
    In(P_HISTORY);
    Out(R(ResourceType::OUT_SIGNAL));
    Emit({Family::REFERENCE, Pass::Copy}, 16, 16, sizeof(ReferenceCopyConstants));
}

void Scheduler::UpdateReference(const DenoiserSlot& slot)
{
    const ReferenceSettings& s = slot.settings.reference;
    const CommonSettings& cs = common_;
    if (memcmp(worldToClip.m, worldToClipPrev.m, sizeof(worldToClip.m)) != 0 || cs.accumulationMode != AccumulationMode::CONTINUE || cs.rectSize[0] != cs.rectSizePrev[0] ||
        cs.rectSize[1] != cs.rectSizePrev[1])
        accumulatedFrameNum_ = 0;
    else
        accumulatedFrameNum_ = std::min(accumulatedFrameNum_ + 1, std::min(s.maxAccumulatedFrameNum, REFERENCE_MAX_HISTORY_FRAME_NUM));

    if (ReferenceAccumulateConstants* c = (ReferenceAccumulateConstants*)Push(slot, RF_ACCUMULATE))
    {
        c->gRectOrigin[0] = cs.rectOrigin[0];
        c->gRectOrigin[1] = cs.rectOrigin[1];
        c->gAccumSpeed = 1.0f / (1.0f + (float)accumulatedFrameNum_);
        c->gDebug = cs.debug;
    }
    if (ReferenceCopyConstants* c = (ReferenceCopyConstants*)Push(slot, RF_COPY))
    {
        c->gRectSizeInv[0] = 1.0f / float(cs.rectSize[0]);
        c->gRectSizeInv[1] = 1.0f / float(cs.rectSize[1]);
        c->gSplitScreen = cs.splitScreen;
    }
}
} // namespace nrdb200

// engine_slots.h -- where the library's subsystems keep their per-engine state.  Host only, not part of the C ABI.
//
// UhcEngine (step_kernel.cu) holds one pointer per subsystem, null until that subsystem attaches its context.  Only the subsystem's own .cu
// file reads or writes its slot, and it nulls the slot when it frees the context; uhc_engine_destroy calls every subsystem's release, so
// no context outlives its engine or is found by a later engine at the same address.
#pragma once
#include "../../include/uhc_b200.h"

enum EngineSlot { SLOT_EVAL, SLOT_TRACK, SLOT_ROLLOUT, SLOT_RENDER, SLOT_RENDER_MESH, SLOT_MESH, SLOT_FLOOR, SLOT_VIDEO, SLOT_COUNT };

void *&engine_slot(UhcEngine *e, EngineSlot s);                 // step_kernel.cu
void *engine_slot(const UhcEngine *e, EngineSlot s);

// Dot-interaction kernel instances for D = 208, 224, 240, 256 (templates and C ABI: interaction.cuh, interaction.cu).
#include "interaction.cuh"

TRB_INTERACTION_GROUP(d208_256, 208)

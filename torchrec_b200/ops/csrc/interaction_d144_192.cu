// Dot-interaction kernel instances for D = 144, 160, 176, 192 (templates and C ABI: interaction.cuh, interaction.cu).
#include "interaction.cuh"

TRB_INTERACTION_GROUP(d144_192, 144)

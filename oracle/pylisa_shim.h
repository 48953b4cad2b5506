// Forced include (-include) for compiling LISA's C++ core (lib/LISA: src/*.cpp and wrappers/wrapper.cpp) unmodified
// into the oracle module oracle/_ref/pylisa.  It changes no arithmetic; it does two things (DESIGN.md section 2):
//
//  * Seeding.  The reference seeds every std::mt19937 from std::random_device, so it cannot replay its own output.
//    After <random>, `random_device` is mapped onto a seed source that hands out base, base + 1, ... in construction
//    order: a MarshallPalmerRain takes one seed when it is built, then each MiniLisa / Lisa the next.  base comes from
//    the environment variable PYLISA_SEED (default 0) and is reset by the exported pylisa_set_seed(base).
//  * Lifetime.  MiniLisa() delegates with the temporaries Lidar(), Water() and MarshallPalmerRain() bound to reference
//    members: GCC rejects it and elsewhere it dangles.  Once Lidar.h, Material.h and ParticleDist.h are in, those three
//    expressions name objects that live for the whole process (one of each, shared by every default-built augmenter).
#ifndef PYLISA_SHIM_H
#define PYLISA_SHIM_H

#include <cstdint>
#include <cstdlib>
#include <random>

namespace pylisa_shim {
inline uint32_t &next_seed()
{
    static uint32_t next = [] {
        const char *s = std::getenv("PYLISA_SEED");
        return s ? (uint32_t)std::strtoul(s, nullptr, 0) : 0u;
    }();
    return next;
}

struct seeded_device {
    typedef unsigned int result_type;
    seeded_device() : value(next_seed()++) {}
    result_type operator()() { return value; }
    static constexpr result_type min() { return 0; }
    static constexpr result_type max() { return 0xffffffffu; }
    double entropy() const noexcept { return 0.0; }
    const result_type value;
};
}  // namespace pylisa_shim

extern "C" __attribute__((visibility("default"), used)) inline void pylisa_set_seed(uint32_t base)
{
    pylisa_shim::next_seed() = base;
}
extern "C" __attribute__((visibility("default"), used)) inline uint32_t pylisa_next_seed() { return pylisa_shim::next_seed(); }

namespace std { using pylisa_seeded_device = pylisa_shim::seeded_device; }
#define random_device pylisa_seeded_device

#include "Lidar.h"
#include "Material.h"
#include "ParticleDist.h"

namespace pylisa_shim {
inline Lidar &default_lidar() { static Lidar *l = new Lidar(); return *l; }
inline Water &default_water() { static Water *w = new Water(); return *w; }
inline MarshallPalmerRain &default_rain() { static MarshallPalmerRain *r = new MarshallPalmerRain(); return *r; }
}  // namespace pylisa_shim

#define Lidar() pylisa_shim::default_lidar()
#define Water() pylisa_shim::default_water()
#define MarshallPalmerRain() pylisa_shim::default_rain()

#endif  // PYLISA_SHIM_H

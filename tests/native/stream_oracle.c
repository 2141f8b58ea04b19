/* Test-side export of the CPU oracle's MT19937 after a scene (tests/explore_oracle.py compiles it with the CPU oracle's
 * flags): oracle/crowdsim_oracle.c is included as it stands, seeded with `seed` and run through its own generate_scene, and
 * the generator's state is returned in numpy's representation (key[624], pos; pos 624 = a full twist comes next). */
#include "../../oracle/crowdsim_oracle.c"

void so_post_generation(const crowdsim_reset_args *a, int N, uint32_t seed, uint32_t *key, int32_t *pos)
{
    double hp[2 * CROWDSIM_MAX_HUMANS], hg[2 * CROWDSIM_MAX_HUMANS], ha[2 * CROWDSIM_MAX_HUMANS];
    mt_state s;
    mt_seed(&s, seed);
    generate_scene(&s, a, N, hp, hg, ha);
    memcpy(key, s.mt, sizeof(s.mt));
    *pos = s.pos;
}

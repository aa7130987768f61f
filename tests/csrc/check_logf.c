// Host check of lz_logf_exact (lightzero_b200/csrc/lz_exact_math.h) against libm logf (the function the reference
// Gumbel tree calls).  usage: check_logf <stride>   (stride 1 = every positive normal float, ~2.1e9 inputs)
// Also checks lz_expf_exact on the inputs the Gumbel read-outs feed it: -inf and every float below -104.
#include <stdio.h>
#include <stdlib.h>
#include "../../lightzero_b200/csrc/lz_exact_math.h"
static inline uint32_t asu32(float f){uint32_t u;memcpy(&u,&f,4);return u;}
static inline float asf(uint32_t u){float f;memcpy(&f,&u,4);return f;}
int main(int argc,char**argv){
  uint32_t stride = argc>1 ? (uint32_t)atoi(argv[1]) : 1;
  unsigned long long bad=0, tot=0;
  for(uint64_t u=0x00800000ull; u<0x7f800000ull; u+=stride){      // positive normal floats
    float x=asf((uint32_t)u); float ref=logf(x), mine=lz_logf_exact(x);
    if(asu32(ref)!=asu32(mine)){ if(bad<10) printf("logf mismatch x=%a ref=%a mine=%a\n",x,ref,mine); bad++; }
    tot++;
  }
  float lspecials[]={1.0f,2.0f,18.0f,82.0f,1.0000001f,0x1.fffffep-1f,0x1p-126f,0x1.fffffep127f};
  for(unsigned i=0;i<sizeof(lspecials)/4;i++){ float x=lspecials[i]; float ref=logf(x), mine=lz_logf_exact(x);
    if(asu32(ref)!=asu32(mine)){ printf("logf special mismatch x=%a ref=%a mine=%a\n",x,ref,mine); bad++; } tot++; }
  // expf below -104 (0xc2d00000) down to -inf: libm returns +0 (or a subnormal) -- the restatement must agree bit for bit
  for(uint64_t u=0xc2d00000ull; u<=0xff800000ull; u+=stride){
    float x=asf((uint32_t)u); float ref=expf(x), mine=lz_expf_exact(x);
    if(asu32(ref)!=asu32(mine)){ if(bad<20) printf("expf mismatch x=%a ref=%a mine=%a\n",x,ref,mine); bad++; }
    tot++;
  }
  { float x=-__builtin_huge_valf(); float ref=expf(x), mine=lz_expf_exact(x);
    if(asu32(ref)!=asu32(mine)){ printf("expf(-inf) mismatch ref=%a mine=%a\n",ref,mine); bad++; } tot++; }
  printf("checked %llu mismatches %llu\n",tot,bad);
  return bad?1:0;
}

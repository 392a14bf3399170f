#include "text.h"
#include <stdio.h>
#include <math.h>
using namespace mg4;
int main(){
  std::mt19937 rng(7);
  // vocabulary: 3 specials + 256 bytes + random pieces
  std::vector<LlamaVocabEntry> v;
  auto add=[&](std::string t,float s){ LlamaVocabEntry e; e.text=t; e.score=s; v.push_back(e); };
  add("<unk>",0); add("<s>",0); add("</s>",0);
  for(int b=0;b<256;++b){ char buf[8]; snprintf(buf,8,"<0x%02X>",b); add(buf,0); }
  for(int i=0;i<3000;++i){ int n=1+rng()%6; std::string t; for(int k=0;k<n;++k) t.push_back((char)(rng()%3? 'a'+rng()%26 : rng()%256)); add(t,-(float)(rng()%1000)/10.f); }
  Tokenizer tk; tk.init(v);
  size_t tot=0;
  for(int it=0;it<20000;++it){ int n=rng()%200; std::string s; for(int k=0;k<n;++k) s.push_back((char)(rng()%4? 'a'+rng()%26 : rng()%256)); auto ids=tk.encode(s,rng()&1); tot+=ids.size(); for(auto id:ids) if(id<0||id>=(int)v.size()) { printf("bad id\n"); return 1; } }
  printf("tokens %zu\n",tot);
  Sampler sm(1); std::vector<float> lg(3259);
  for(int it=0;it<20000;++it){
    int mode=rng()%6;
    for(auto&x:lg){ x=(float)((int)(rng()%2000)-1000)/50.f; }
    if(mode==1) for(int k=0;k<10;++k) lg[rng()%lg.size()]=INFINITY;
    if(mode==2) for(int k=0;k<10;++k) lg[rng()%lg.size()]=-INFINITY;
    if(mode==3) for(int k=0;k<10;++k) lg[rng()%lg.size()]=NAN;
    if(mode==4) for(auto&x:lg) x=0;
    SamplingArgs p{ (float)(rng()%300)/100.f-0.2f, (int)(rng()%100)-10, (float)(rng()%120)/100.f, (float)(rng()%120)/100.f, (float)(rng()%120)/100.f, (int)(rng()%3), (float)(rng()%100)/10.f, (float)(rng()%100)/100.f };
    int id=sm.sample(lg.data(),(int)lg.size(),p);
    if(id<0||id>=(int)lg.size()){ printf("bad sample id %d mode %d\n",id,mode); return 1; }
  }
  printf("sampler ok\n"); return 0; }
